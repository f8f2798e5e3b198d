"""Time per-clip sampling controls of the body prior on an H100 against scalar calls.

One batch of B clips whose clips need four different settings (sampled at 0.8, greedy, top-k 64 + top-p 0.9, min-p 0.05 at
1.3), at 64 x 75 and 12 x 75 (clips x latent rows) on the dim 256 prior and at 64 x 75 on the 6-D (dim 512) prior, the
variants alternating inside one run, noise drawn outside the timed region:
  (a) default: the default draw of the whole batch (the default sampler kernels);
  (b) warp: one scalar call of the whole batch at temperature 0.8 (the sampler kernels that also serve per-clip calls);
  (c) clips: one per-clip call of the whole batch, clip b taking setting b % 4;
  (d) four: the same four groups of clips as four scalar calls, one per setting, each on its own clips.
Every variant is ``Engine.body_generate`` (audio encoder, sampler, both VQ decoders) and is timed with CUDA events around
all of its calls after warm-up; the median and the range are reported with the card's name, power limit and SM clocks read
in the same run.  Prints one JSON line per shape.

    python bench_clip_ctl.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json

import torch

from bench_seeded import card, timed
from talkshow_b200 import synth
from talkshow_b200.engine import Engine

SHAPES = [("3d", 64, 75), ("3d", 12, 75), ("6d", 64, 75)]
GROUPS = [dict(temperature=0.8), dict(temperature=0.0), dict(temperature=1.0, top_k=64, top_p=0.9),
          dict(temperature=1.3, min_p=0.05)]


def per_clip(B):
    """the four settings as per-clip lists: clip b takes GROUPS[b % 4]"""
    full = [dict(dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0), **GROUPS[b % 4]) for b in range(B)]
    return {k: [c[k] for c in full] for k in ("temperature", "top_k", "top_p", "min_p")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip_ctl.py needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    engines = {}
    for geo, B, T in SHAPES:
        if geo not in engines:
            six = geo == "6d"
            ck = synth.body_pixel_checkpoint_6d(0) if six else synth.body_pixel_checkpoint(0)
            vq = synth.body_vq_checkpoint_6d(0) if six else synth.body_vq_checkpoint(0)
            e = Engine(0)
            e.load_pixelcnn(ck["generator"])
            e.load_audioenc(ck["audioencoder"])
            e.load_vq(0, vq["g_body"])
            e.load_vq(1, vq["g_hand"])
            engines[geo] = e
        e = engines[geo]
        mfcc = synth.synth_mfcc(B, 4 * T, seed=7).cuda()
        label = (torch.arange(B) % 4).cuda()
        noise = torch.empty(2 * T, B, 2048, device=dev).exponential_(1)
        pc = per_clip(B)
        groups = []
        for g, s in enumerate(GROUPS):
            idx = torch.arange(g, B, 4, device=dev)
            groups.append((mfcc[idx].contiguous(), label[idx].contiguous(),
                           noise[:, idx].contiguous() if s["temperature"] > 0 else None, s))

        def four():
            for m, lab, nz, s in groups:
                e.body_generate(m, lab, nz, **s)

        settings = {
            "a_default": lambda: e.body_generate(mfcc, label, noise),
            "b_warp": lambda: e.body_generate(mfcc, label, noise, temperature=0.8),
            "c_clips": lambda: e.body_generate(mfcc, label, noise, **pc),
            "d_four": four,
        }
        med, rng = timed(settings, args.warmup, args.iters)
        print(json.dumps({"bench": "clip_ctl", "call": "Engine.body_generate", "prior": geo, "B": B, "T": T,
                          "median_ms": med, "range_ms": rng, "iters": args.iters, **card()}), flush=True)
    torch.cuda.synchronize()
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
