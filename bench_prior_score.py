"""Time Engine.pixelcnn_score (time-parallel teacher-forced PixelCNN + cross-entropy) against the sequential teacher-forced
path Engine.pixelcnn_logits at the benchmark shape (64 clips x 10 s, T = 75 latent rows) and at 12 clips, on an H100.
The two calls alternate inside one run, timed with CUDA events after warm-up.  Prints one JSON line.

    python bench_prior_score.py [--iters 20] [--warmup 3]

Achieved rate: 69,337,088 FLOP per latent row per sample (BASELINE.md section 4: every dense layer of the dim 256 x 15
prior, both columns) over the score call's time, against the fp32-grade peak of the fp16-split wgmma kernel, 989 / 3
TFLOP/s (three fp16 products per fp32-grade multiply-add, H100 SXM data sheet).  Needs a GPU; writes nothing."""
import argparse
import json
import subprocess

import torch

from talkshow_b200 import synth
from talkshow_b200.engine import Engine

FLOP_PER_ROW = 69_337_088
PEAK_TFLOPS = 989.0 / 3


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit": q[1]}


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prior_score.py needs a CUDA device")
    torch.set_grad_enabled(False)
    ck = synth.body_pixel_checkpoint(0)
    e = Engine(0)
    e.load_pixelcnn(ck["generator"])
    out = {"metric": "prior_score_ms", "flop_per_row": FLOP_PER_ROW, "peak_tflops_fp32_grade": round(PEAK_TFLOPS, 1)}
    out.update(card())
    g = torch.Generator().manual_seed(0)
    for B in (64, 12):
        T = 75
        aud = (torch.randn(B, 256, T, generator=g) * 0.5).cuda()
        label = (torch.arange(B) % 4).cuda()
        codes = torch.randint(0, 2048, (B, T, 2), generator=g).cuda()
        score = lambda: e.pixelcnn_score(aud, label, codes)        # noqa: E731
        seq = lambda: e.pixelcnn_logits(aud, label, codes)         # noqa: E731
        for _ in range(args.warmup):
            score()
            seq()
        torch.cuda.synchronize()
        n0 = e.launches
        score()
        n_score = e.launches - n0
        n0 = e.launches
        seq()
        n_seq = e.launches - n0
        ms_score, ms_seq = [], []
        for _ in range(args.iters):          # alternate the two paths so drift hits both alike
            ms_score.append(timed(score, 1))
            ms_seq.append(timed(seq, 1))
        ms_score.sort()
        ms_seq.sort()
        s_med, q_med = ms_score[len(ms_score) // 2], ms_seq[len(ms_seq) // 2]
        tflops = FLOP_PER_ROW * B * T / (s_med * 1e-3) / 1e12
        out["b%d_t%d" % (B, T)] = {
            "score_ms": round(s_med, 3), "score_ms_min": round(ms_score[0], 3),
            "logits_sequential_ms": round(q_med, 3), "logits_sequential_ms_min": round(ms_seq[0], 3),
            "speedup": round(q_med / s_med, 2), "score_tflops_fp32_grade": round(tflops, 1),
            "score_share_of_peak": round(tflops / PEAK_TFLOPS, 3),
            "launches_score": n_score, "launches_sequential": n_seq}
    e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
