"""Time seeded sampling of the body prior on an H100 against the noise-tensor paths it replaces.

One ``Engine.body_generate`` call per setting, the settings alternating inside one run, at 64 x 75, 12 x 75 and 1 x 30
(clips x latent rows) on the dim 256 prior and at 64 x 75 on the 6-D (dim 512) prior:
  (a) explicit: noise drawn outside the timed region (the sampler alone);
  (b) per-step: ``draw_sampler_noise(per_step=True)`` inside the timed region (2T exponential_ calls, what the wrappers do
      by default);
  (c) batched: one ``exponential_`` of [2T,B,2048] inside the timed region (what bench.py does);
  (d) seeded: ``seeds=`` (ts_body_sample_seeded), no noise tensor.
Then one ``WholeBody.generate`` at 64 clips x 10 s with (b) and with (d).  Each call is timed with CUDA events after
warm-up; the median and the range are reported with the noise bytes each call avoids (computed from the shapes), and the
card's name, power limit and SM clocks read in the same run.  Prints one JSON line per shape.

    python bench_seeded.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json
import statistics
import subprocess

import torch

from talkshow_b200 import synth
from talkshow_b200.engine import Engine, clip_seeds
from talkshow_b200.nets.base import draw_sampler_noise

SHAPES = [("3d", 64, 75), ("3d", 12, 75), ("3d", 1, 30), ("6d", 64, 75)]


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit": q[1], "sm_clock": q[2], "sm_clock_max": q[3]}


def timed(settings, warmup, iters):
    times = {n: [] for n in settings}
    for it in range(warmup + iters):
        for n, fn in settings.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if it >= warmup:
                times[n].append(a.elapsed_time(b))
    return ({n: round(statistics.median(v), 3) for n, v in times.items()},
            {n: round(max(v) - min(v), 3) for n, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seeded.py needs a CUDA device")
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    ckpts = {}
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
            engines[geo], ckpts[geo] = e, (ck, vq)
        e = engines[geo]
        mfcc = synth.synth_mfcc(B, 4 * T, seed=7).cuda()
        label = (torch.arange(B) % 4).cuda()
        noise = torch.empty(2 * T, B, 2048, device=dev).exponential_(1)
        seeds = clip_seeds(1234, B).cuda()
        settings = {
            "a_explicit": lambda: e.body_generate(mfcc, label, noise),
            "b_per_step": lambda: e.body_generate(mfcc, label, draw_sampler_noise(T, B, dev, per_step=True)),
            "c_batched": lambda: e.body_generate(mfcc, label, draw_sampler_noise(T, B, dev, per_step=False)),
            "d_seeded": lambda: e.body_generate(mfcc, label, None, seeds=seeds),
        }
        med, rng = timed(settings, args.warmup, args.iters)
        print(json.dumps({"bench": "seeded", "call": "Engine.body_generate", "prior": geo, "B": B, "T": T,
                          "median_ms": med, "range_ms": rng, "noise_bytes_avoided": 2 * T * B * 2048 * 4,
                          "iters": args.iters, **card()}), flush=True)
    # the whole-body call at 64 clips x 10 s: face + body + assembly, default noise against seeded
    from talkshow_b200.pipeline import WholeBody

    ck, vq = ckpts["3d"]
    wb = WholeBody(Engine(0))
    wb.load(ck, vq, synth.face_checkpoint(0))
    B, M = 64, 300
    T = M // 4
    mfcc = synth.synth_mfcc(B, M, seed=8).cuda()
    wave = torch.randn(B, 16000 * 10, generator=torch.Generator().manual_seed(9)).cuda()
    label = (torch.arange(B) % 4).cuda()
    settings = {"b_per_step": lambda: wb.generate(mfcc, wave, label),
                "d_seeded": lambda: wb.generate(mfcc, wave, label, clip_seeds=1234)}
    med, rng = timed(settings, args.warmup, args.iters)
    print(json.dumps({"bench": "seeded", "call": "WholeBody.generate", "prior": "3d", "B": B, "T": T, "seconds": 10,
                      "median_ms": med, "range_ms": rng, "noise_bytes_avoided": 2 * T * B * 2048 * 4,
                      "iters": args.iters, **card()}), flush=True)
    torch.cuda.synchronize()
    wb.close()
    wb.e.close()
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
