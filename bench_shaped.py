"""Time logit shaping of the body prior (repetition penalty and code bias) on an H100 against the unshaped sampler call.

At 64 x 75, 12 x 75 and 1 x 30 (clips x latent rows) on the dim-256 prior with the grid-wide executor (mode 0) and the
cluster executor (mode 2), and on the 6-D (dim 512) prior with the cluster executor, the variants alternating inside one
run, noise drawn outside the timed region:
  (a) warp: the unshaped call at temperature 0.8 (the sampler kernels that also serve shaped calls);
  (b) w8: repetition penalty 1.5 over a window of 8 rows;
  (c) wall: repetition penalty 1.5 over a window covering the whole clip;
  (d) w8_bias / (e) wall_bias: (b) / (c) with a code bias that bans 512 codes of every row.
Every variant is ``Engine.pixelcnn_generate`` (sampler only: three audio GEMMs and the sampler kernel) and is timed with
CUDA events around the call after warm-up; the median and the range are reported with the card's name, power limit and
SM clocks read in the same run.  Prints one JSON line per shape and executor.

    python bench_shaped.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json

import torch

from bench_seeded import card, timed
from talkshow_b200 import synth
from talkshow_b200.engine import Engine

SHAPES = [("3d", 0, 64, 75), ("3d", 0, 12, 75), ("3d", 0, 1, 30), ("3d", 2, 64, 75), ("3d", 2, 12, 75), ("3d", 2, 1, 30),
          ("6d", 2, 64, 75), ("6d", 2, 12, 75), ("6d", 2, 1, 30)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shaped.py needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    engines = {}
    for geo, mode, B, T in SHAPES:
        if geo not in engines:
            ck = synth.body_pixel_checkpoint_6d(0) if geo == "6d" else synth.body_pixel_checkpoint(0)
            e = Engine(0)
            e.load_pixelcnn(ck["generator"])
            e.load_audioenc(ck["audioencoder"])
            engines[geo] = e
        e = engines[geo]
        e.set_pixelcnn_mode(mode)
        mfcc = synth.synth_mfcc(B, 4 * T, seed=7).cuda()
        aud = e.audio_encode(mfcc)
        label = (torch.arange(B) % 4).cuda()
        noise = torch.empty(2 * T, B, 2048, device=dev).exponential_(1)
        g = torch.Generator(device=dev).manual_seed(8)
        bias = torch.zeros(B, 2, 2048, device=dev)
        bias.scatter_(-1, torch.rand(B, 2, 2048, device=dev, generator=g).argsort(-1)[..., :512], float("-inf"))
        run = lambda **kw: e.pixelcnn_generate(aud, label, noise, temperature=0.8, **kw)
        settings = {
            "a_warp": lambda: run(),
            "b_w8": lambda: run(repetition_penalty=1.5, repetition_window=8),
            "c_wall": lambda: run(repetition_penalty=1.5, repetition_window=T),
            "d_w8_bias": lambda: run(repetition_penalty=1.5, repetition_window=8, code_bias=bias),
            "e_wall_bias": lambda: run(repetition_penalty=1.5, repetition_window=T, code_bias=bias),
        }
        # the bias check (one device read-back) is part of the call a user makes; time it as such
        med, rng = timed(settings, args.warmup, args.iters)
        print(json.dumps({"bench": "shaped", "call": "Engine.pixelcnn_generate", "prior": geo, "executor": mode, "B": B,
                          "T": T, "median_ms": med, "range_ms": rng, "iters": args.iters, **card()}), flush=True)
    torch.cuda.synchronize()
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
