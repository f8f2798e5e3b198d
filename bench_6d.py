"""Time pipeline.WholeBody.generate on convert_to_6d synthetic checkpoints (identity-free 6-D face, dim 512 x 10-layer prior,
78 / 180-channel VQ decoders, fused 6-D assembly) on an H100, with CUDA events after warm-up.  Shapes: 64 clips x 10 s,
12 x 10 s and 1 x 4 s.  At 64 x 10 s the 3-D WholeBody (shipped geometry, with its side-by-side sampler engine) runs in
alternation with the 6-D one, for context.  Prints one JSON line per shape with the card's name and power limit.

    python bench_6d.py [--steps 10] [--warmup 2]

ms_per_step is one generate call (face + body + assembly, device time between events around the call);
frames_per_s = clips x frames / step time; sampler_ms is the PixelCNN sampler's own device time inside that call
(Engine.pixelcnn_last_ms, median over the timed steps).  Needs a GPU; writes nothing."""
import argparse
import json
import subprocess

import torch

from talkshow_b200 import synth
from talkshow_b200.engine import Engine
from talkshow_b200.pipeline import WholeBody

SHAPES = ((64, 10), (12, 10), (1, 4))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit": q[1]}


def inputs(B, sec, T):
    wave = synth.synth_wave(B, 16000 * sec, seed=B + sec).cuda()
    mfcc = synth.synth_mfcc(B, 30 * sec, seed=B + sec).cuda()
    label = (torch.arange(B) % 4).cuda()
    noise = torch.empty(2 * T, B, 2048).exponential_(1, generator=torch.Generator().manual_seed(B)).cuda()
    return mfcc, wave, label, noise


def step(wb, x):
    """one generate call between two events -> (ms, sampler ms)"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    wb.generate(*x[:3], noise=x[3])
    b.record()
    b.synchronize()
    return a.elapsed_time(b), wb.pixelcnn_last_ms()


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_6d.py needs a CUDA device")
    torch.set_grad_enabled(False)
    info = card()
    wb6 = WholeBody(Engine(0))
    wb6.load(synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0), synth.face_checkpoint_6d(0))
    wb6.pixelcnn_timing(True)
    wb3 = WholeBody(Engine(0))
    wb3.load(synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), synth.face_checkpoint(0))
    wb3.pixelcnn_timing(True)
    for B, sec in SHAPES:
        x = inputs(B, sec, wb6.e.latent_rows(30 * sec))
        runs = [("6d", wb6)] + ([("3d", wb3)] if (B, sec) == (64, 10) else [])
        for _ in range(args.warmup):
            for _, wb in runs:
                step(wb, x)
        ms = {k: [] for k, _ in runs}
        smp = {k: [] for k, _ in runs}
        for _ in range(args.steps):          # alternate the two geometries so drift hits both alike
            for k, wb in runs:
                t, s = step(wb, x)
                ms[k].append(t)
                smp[k].append(s)
        frames = B * 30 * sec
        out = {"metric": "whole_body_6d_ms_per_step", "clips": B, "seconds": sec, "frames": frames, "steps": args.steps}
        out.update(info)
        for k, _ in runs:
            pre = "" if k == "6d" else "3d_"
            out[pre + "ms_per_step"] = round(median(ms[k]), 3)
            out[pre + "ms_per_step_min"] = round(min(ms[k]), 3)
            out[pre + "frames_per_s"] = round(frames / (median(ms[k]) * 1e-3), 1)
            out[pre + "sampler_ms"] = round(median(smp[k]), 3)
        print(json.dumps(out), flush=True)
    torch.cuda.synchronize()
    wb3.close()
    wb6.close()
    wb3.e.close()
    wb6.e.close()


if __name__ == "__main__":
    main()
