"""Time guided sampling of the body prior on an H100 against the unguided sampler call.

At 64 x 75, 12 x 75 and 1 x 30 (clips x latent rows) on the dim-256 prior with the grid-wide executor (mode 0), at 64 x 75
with the cluster executor (mode 2), and at 64 x 75 on the 6-D (dim 512) prior with the cluster executor, the settings
alternating inside one run, noise drawn outside the timed region:
  (a) warp_B: the unguided call at temperature 0.8 on the B clips (the sampler kernels that also serve guided calls);
  (b) guided_w1: the guided call at w = 1 against silence (2B branches);
  (c) guided_w2: the guided call at w = 2 against silence;
  (d) warp_2B: the unguided call at temperature 0.8 on 2B clips.
Every setting is one ``Engine.body_generate`` (audio encoder, sampler and the two VQ decoders; the guided calls encode
both branches and decode the B clips) timed with CUDA events around the call after warm-up; the median and the range are
reported with the card's name, power limit and SM clocks read in the same run.  At 64 clips the grid-wide executor runs
the guided call as two launches of 64 branches.  Prints one JSON line per shape and executor.

    python bench_guided.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json

import torch

from bench_seeded import card, timed
from talkshow_b200 import synth
from talkshow_b200.engine import Engine

SHAPES = [("3d", 0, 64, 75), ("3d", 0, 12, 75), ("3d", 0, 1, 30), ("3d", 2, 64, 75), ("6d", 2, 64, 75)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_guided.py needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    engines = {}
    for geo, mode, B, T in SHAPES:
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
        e.set_pixelcnn_mode(mode)
        M = 4 * T
        mfcc = synth.synth_mfcc(2 * B, M, seed=7).cuda()
        label = (torch.arange(2 * B) % 4).cuda()
        sil = e.silence_mfcc(M, B)
        noise = torch.empty(2 * T, 2 * B, 2048, device=dev).exponential_(1)
        nB = noise[:, :B].contiguous()
        run = lambda n, **kw: e.body_generate(mfcc[:n], label[:n], noise if n == 2 * B else nB, temperature=0.8, **kw)
        settings = {
            "a_warp_B": lambda: run(B),
            "b_guided_w1": lambda: run(B, guidance=1.0, guide_mfcc=sil),
            "c_guided_w2": lambda: run(B, guidance=2.0, guide_mfcc=sil),
            "d_warp_2B": lambda: run(2 * B),
        }
        med, rng = timed(settings, args.warmup, args.iters)
        print(json.dumps({"bench": "guided", "call": "Engine.body_generate", "prior": geo, "executor": mode, "B": B, "T": T,
                          "median_ms": med, "range_ms": rng, "iters": args.iters, **card()}), flush=True)
    torch.cuda.synchronize()
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
