"""Time the body prior's sampler under nucleus (top-p) and min-p sampling on an H100: the default draw
(ts_pixelcnn_generate) against top-k 50 (ts_pixelcnn_sample), top-p 0.9, top-k 50 with top-p 0.9, and min-p 0.05
(ts_pixelcnn_sample_ctl), all at temperature 1, at 64 x 75, 12 x 75 and 1 x 30 (clips x latent rows) on the dim 256 prior
and at 64 x 75 on the 6-D (dim 512) prior.  The noise is drawn outside the timed region.  The five settings alternate
inside one run; each call is timed with CUDA events after warm-up and the median is reported.  The card's name, power
limit and SM clocks are read in the same run.  Prints one JSON line per shape, then runs bench.py once (the default
whole-body step, which does not use the controls) and passes its result line through.

    python bench_nucleus.py [--iters 7] [--warmup 2] [--no-step]

Needs a GPU; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

from talkshow_b200 import synth
from talkshow_b200.engine import Engine

# (top_k, top_p, min_p) at temperature 1
SETTINGS = {"default": None, "k50": (50, 1.0, 0.0), "p0.9": (0, 0.9, 0.0), "k50+p0.9": (50, 0.9, 0.0), "m0.05": (0, 1.0, 0.05)}
SHAPES = [("3d", 64, 75), ("3d", 12, 75), ("3d", 1, 30), ("6d", 64, 75)]


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit": q[1], "sm_clock": q[2], "sm_clock_max": q[3]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-step", action="store_true", help="skip the bench.py run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nucleus.py needs a CUDA device")
    torch.set_grad_enabled(False)
    engines = {}
    for geo, B, T in SHAPES:
        if geo not in engines:
            ck = synth.body_pixel_checkpoint_6d(0) if geo == "6d" else synth.body_pixel_checkpoint(0)
            e = Engine(0)
            e.load_pixelcnn(ck["generator"])
            e.load_audioenc(ck["audioencoder"])
            engines[geo] = e
        e = engines[geo]
        aud = e.audio_encode(synth.synth_mfcc(B, 4 * T, seed=7).cuda())
        label = (torch.arange(B) % 4).cuda()
        noise = torch.empty(2 * T, B, 2048, device="cuda").exponential_(1)

        def run(s):
            if s is None:
                return e.pixelcnn_generate(aud, label, noise)
            k, p, m = s
            return e.pixelcnn_generate(aud, label, noise, top_k=k, top_p=p, min_p=m)

        times = {n: [] for n in SETTINGS}
        for it in range(args.warmup + args.iters):
            for n, s in SETTINGS.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                run(s)
                b.record()
                b.synchronize()
                if it >= args.warmup:
                    times[n].append(a.elapsed_time(b))
        med = {n: round(statistics.median(v), 3) for n, v in times.items()}
        spread = {n: round(max(v) - min(v), 3) for n, v in times.items()}
        print(json.dumps({"bench": "nucleus", "prior": geo, "B": B, "T": T, "median_ms": med, "range_ms": spread,
                          "iters": args.iters, **card()}), flush=True)
    for e in engines.values():
        e.close()
    if not args.no_step:
        here = os.path.dirname(os.path.abspath(__file__))
        subprocess.run([sys.executable, os.path.join(here, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3", "--no-cpu-baseline", "--no-extras"], check=True)


if __name__ == "__main__":
    main()
