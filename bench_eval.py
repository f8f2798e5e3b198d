"""Time held-out scoring on an H100: pipeline.WholeBody.evaluate and its three parts, with CUDA events after warm-up, for
the 3-D and the convert_to_6d ("6-D") synthetic trios at 64 clips x 10 s and 12 clips x 10 s.  Prints one JSON line per
shape with the card's name, power limit and the SM clock read during the run.

    python bench_eval.py [--steps 10] [--warmup 2]

Per geometry (the two alternate step by step, so drift hits both alike):
  <g>_ms        one WholeBody.evaluate call (face score, VQ score of the pair, audio encoder + prior score, the host-side
                loss reductions included), device time between events around the call, median over the steps;
  <g>_face_ms   Engine.face_score alone;  <g>_vq_ms  Engine.vq_score of body and hands;
  <g>_prior_ms  Engine.audio_encode + Engine.pixelcnn_score on the VQ codes.
Needs a GPU; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests", "golden"))

from make_golden_eval import synth_expression  # noqa: E402
from talkshow_b200 import synth  # noqa: E402
from talkshow_b200.data_utils.lower_body import c_index_3d, c_index_6d  # noqa: E402
from talkshow_b200.engine import Engine  # noqa: E402
from talkshow_b200.pipeline import WholeBody  # noqa: E402

SHAPES = ((64, 10), (12, 10))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit": q[1], "sm_clock": q[2], "sm_clock_max": q[3]}


def batch(six, B, sec):
    nf = 30 * sec
    poses = synth.synth_poses(B, nf, seed=B)
    if six:
        poses = torch.cat([poses, synth.synth_poses(B, nf, seed=B + 1)], 1)
    return {"wave": synth.synth_wave(B, 16000 * sec, seed=B).cuda(), "aud_feat": synth.synth_mfcc(B, nf, seed=B).cuda(),
            "poses": poses.cuda(), "expression": synth_expression(B, nf, B).cuda(), "speaker": (20 + torch.arange(B) % 4).cuda()}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def parts(wb, six, bat):
    """the three parts of evaluate as separate callables over device tensors prepared once"""
    e = wb.e
    label = bat["speaker"] - 20
    idv = torch.nn.functional.one_hot(label, 4).float()
    gt_face = torch.cat([bat["poses"].permute(0, 2, 1), bat["expression"].permute(0, 2, 1)], 2).contiguous()
    gt = bat["poses"][:, c_index_6d if six else c_index_3d].permute(0, 2, 1)
    nb = 78 if six else 39
    pb, ph = gt[..., :nb].contiguous(), gt[..., nb:].contiguous()
    codes = torch.stack([e.vq_encode(0, pb), e.vq_encode(1, ph)], -1)
    return {"face": lambda: e.face_score(bat["wave"], idv, gt_face),
            "vq": lambda: (e.vq_score(0, pb), e.vq_score(1, ph)),
            "prior": lambda: e.pixelcnn_score(e.audio_encode(bat["aud_feat"]), label, codes)}


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    torch.set_grad_enabled(False)
    wbs = {}
    for g, (face, vq, bp) in (("3d", (synth.face_checkpoint(0), synth.body_vq_checkpoint(0), synth.body_pixel_checkpoint(0))),
                              ("6d", (synth.face_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0),
                                      synth.body_pixel_checkpoint_6d(0)))):
        wbs[g] = WholeBody(Engine(0), overlap_batch=0)
        wbs[g].load(bp, vq, face)
    for B, sec in SHAPES:
        runs = {}
        for g, wb in wbs.items():
            bat = batch(g == "6d", B, sec)
            fns = {"": lambda wb=wb, bat=bat: wb.evaluate(bat)}
            fns.update({"_" + k: f for k, f in parts(wb, g == "6d", bat).items()})
            runs[g] = fns
        for _ in range(args.warmup):
            for fns in runs.values():
                for f in fns.values():
                    timed(f)
        ms = {(g, k): [] for g, fns in runs.items() for k in fns}
        for _ in range(args.steps):
            for g, fns in runs.items():
                for k, f in fns.items():
                    ms[(g, k)].append(timed(f))
        out = {"metric": "evaluate_ms", "clips": B, "seconds": sec, "frames": B * 30 * sec, "steps": args.steps}
        out.update(card())
        for (g, k), v in ms.items():
            out["%s%s_ms" % (g, k)] = round(median(v), 3)
        print(json.dumps(out), flush=True)
    torch.cuda.synchronize()
    for wb in wbs.values():
        wb.close()
        wb.e.close()


if __name__ == "__main__":
    main()
