"""Time the body prior's sampler under its sampling controls on an H100: the default draw (ts_pixelcnn_generate) against
temperature 0.8, top-k 50 at temperature 1, and greedy decoding (ts_pixelcnn_sample), at 64 x 75, 12 x 75 and 1 x 30
(clips x latent rows) on the dim 256 prior and at 64 x 75 on the 6-D (dim 512) prior.  The four settings alternate inside
one run; each call is timed with CUDA events after warm-up and the median is reported.  The card's name, power limit
and SM clocks are read in the same run.  Prints one JSON line per shape.

    python bench_sampling.py [--iters 7] [--warmup 2]

Needs a GPU; writes nothing."""
import argparse
import json
import statistics
import subprocess

import torch

from talkshow_b200 import synth
from talkshow_b200.engine import Engine

SETTINGS = {"default": None, "t0.8": (0.8, 0), "k50": (1.0, 50), "greedy": (0.0, 0)}
SHAPES = [("3d", 64, 75), ("3d", 12, 75), ("3d", 1, 30), ("6d", 64, 75)]


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit": q[1], "sm_clock": q[2], "sm_clock_max": q[3]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py needs a CUDA device")
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
            t, k = s
            return e.pixelcnn_generate(aud, label, None if t == 0 else noise, temperature=t, top_k=k)

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
        print(json.dumps({"bench": "sampling", "prior": geo, "B": B, "T": T, "median_ms": med, "range_ms": spread,
                          "iters": args.iters, **card()}), flush=True)
    for e in engines.values():
        e.close()


if __name__ == "__main__":
    main()
