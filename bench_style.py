"""Time styled sampling of the body prior on an H100 against the same unstyled calls.

One ``Engine.body_generate`` call per setting, the settings alternating inside one run, at 64 x 75 and 1 x 30 (clips x
latent rows) on the dim 256 prior and at 64 x 75 on the 6-D (dim 512) prior, noise drawn outside the timed region:
  (a) default: the unstyled default draw (the default sampler kernels);
  (b) warp: the unstyled call with anchors all -1, which runs the sampler kernels that also serve styled calls;
  (c) blend: a per-clip mixture of two speakers ([B, 4] weights, broadcast over the rows);
  (d) fade: a per-row schedule fading from one speaker to another over the middle half of the clip.
The schedules are device tensors, so (c) and (d) include the one synchronisation of the value check a user pays.  Each
call is timed with CUDA events after warm-up; the median and the range are reported with the card's name, power limit and
SM clocks read in the same run.  Prints one JSON line per shape.

    python bench_style.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json

import torch

from bench_seeded import card, timed
from talkshow_b200 import synth
from talkshow_b200.engine import Engine

SHAPES = [("3d", 64, 75), ("3d", 1, 30), ("6d", 64, 75)]


def schedules(B, T, dev):
    a, b = torch.arange(B) % 4, (torch.arange(B) + 1) % 4
    blend = 0.5 * torch.nn.functional.one_hot(a, 4).float() + 0.5 * torch.nn.functional.one_hot(b, 4).float()
    t = ((torch.arange(T, dtype=torch.float64) - T // 4) / max(1, T // 2)).clamp(0, 1)[None, :, None]
    fade = (1 - t) * torch.nn.functional.one_hot(a, 4).double()[:, None] + t * torch.nn.functional.one_hot(b, 4).double()[:, None]
    return blend.to(dev), fade.float().to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_style.py needs a CUDA device")
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
        free = torch.full((B, T, 2), -1, dtype=torch.int64, device=dev)
        blend, fade = schedules(B, T, dev)
        settings = {
            "a_default": lambda: e.body_generate(mfcc, label, noise),
            "b_warp": lambda: e.body_generate(mfcc, label, noise, anchors=free),
            "c_blend": lambda: e.body_generate(mfcc, None, noise, style=blend),
            "d_fade": lambda: e.body_generate(mfcc, None, noise, style=fade),
        }
        med, rng = timed(settings, args.warmup, args.iters)
        print(json.dumps({"bench": "style", "call": "Engine.body_generate", "prior": geo, "B": B, "T": T,
                          "median_ms": med, "range_ms": rng, "iters": args.iters, **card()}), flush=True)
    torch.cuda.synchronize()
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
