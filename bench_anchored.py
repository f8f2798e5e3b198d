"""Time anchored sampling of the body prior on an H100 against the same unanchored call.

One ``Engine.body_generate`` call per setting, the settings alternating inside one run, at 64 x 75, 12 x 75 and 1 x 30
(clips x latent rows) on the dim 256 prior and at 64 x 75 on the 6-D (dim 512) prior, noise drawn outside the timed region:
  (a) default: the default draw (the default sampler kernels, no controls);
  (b) warp: the unanchored call with per-draw log p, which runs the sampler kernels that also serve anchored calls;
  (c) half: (b) with a random half of the draws pinned;
  (d) window: (b) with every draw pinned except a free 2 s window (15 latent rows) in the middle of the clip.
The anchors are device tensors, so (c) and (d) include the one synchronisation of the value check a user pays.  Each call is timed with CUDA events after warm-up; the median and the range are reported with the card's name, power
limit and SM clocks read in the same run.  Prints one JSON line per shape.

    python bench_anchored.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json

import torch

from bench_seeded import SHAPES, card, timed
from talkshow_b200 import synth
from talkshow_b200.engine import Engine


def anchors_for(codes, kind, seed):
    B, T, _ = codes.shape
    if kind == "half":
        g = torch.Generator(device=codes.device).manual_seed(seed)
        return torch.where(torch.rand(B, T, 2, generator=g, device=codes.device) < 0.5, codes, -1)
    a = codes.clone()
    lo = max(0, T // 2 - 7)
    a[:, lo:lo + 15] = -1
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_anchored.py needs a CUDA device")
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
        codes = e.body_generate(mfcc, label, noise)[0]
        half, window = anchors_for(codes, "half", 11), anchors_for(codes, "window", 0)
        settings = {
            "a_default": lambda: e.body_generate(mfcc, label, noise),
            "b_warp": lambda: e.body_generate(mfcc, label, noise, want_logp=True),
            "c_half": lambda: e.body_generate(mfcc, label, noise, want_logp=True, anchors=half),
            "d_window": lambda: e.body_generate(mfcc, label, noise, want_logp=True, anchors=window),
        }
        med, rng = timed(settings, args.warmup, args.iters)
        print(json.dumps({"bench": "anchored", "call": "Engine.body_generate", "prior": geo, "B": B, "T": T,
                          "pinned_half": int((half >= 0).sum()), "pinned_window": int((window >= 0).sum()),
                          "median_ms": med, "range_ms": rng, "iters": args.iters, **card()}), flush=True)
    torch.cuda.synchronize()
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
