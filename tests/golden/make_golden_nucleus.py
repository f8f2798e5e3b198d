"""Generate tests/golden/sampling_p.npz: codes and poses of the UNMODIFIED reference's s2g_body_pixel.infer_on_audio
(nets/smplx_body_pixel.py:232-289) under nucleus (top-p) and min-p sampling.  Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_nucleus.py

The recipe is that of make_golden_sampling.py: the module's ``F`` is swapped for a proxy whose ``softmax`` applies the
warp of ts_pixelcnn_sample_ctl (include/talkshow_b200.h) to the raw logits, here stated on its own in numpy:
  - top_k and temperature t as in make_golden_sampling.py; e = exp(l / t - max l / t) in fp32 over the top-k set;
  - integer masses w = rint(e 2^32); top_p keeps code i iff the mass of the codes with a greater logit, A_i, satisfies
    (double)A_i < (double)(float)top_p * (double)sum(w);
  - min_p keeps code i iff e_i >= (float)min_p;
  - the probabilities are the softmax of l / t over the final keep set.
Everything else (the loop, the multinomial draw under the seed, the VQ decoders) is the reference's own code.

The CPU's exp and the GPU's expf differ in the last bit, so a keep set can differ between them only where a boundary lies
within rounding of the threshold.  The script records, per draw, min_i |A_i - P| / W over the codes with A_i > 0 (the
most likely code has A = 0 in any arithmetic and is always kept) and min_i |e_i - m| / m.  A run whose smallest margin is
below MIN_MARGIN is repeated under the next seed (seed + 100, ...), so no keep set of the fixture is ambiguous; the seed
each setting ended on and the smallest margins are stored.  The setting with top_p = 1e-6 must decode greedily: the
script asserts that its codes equal a greedy run and that no draw of it has an exact tie of the maximum logit.  Running
the script again reproduces the file byte for byte (fixed seeds, CPU, one thread).
"""
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.nn.functional as TF  # noqa: E402

from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

SEED = 4100
POSE_STRIDE = 5   # poses are kept for every 5th frame (the codes, which determine them, are kept whole)
MIN_MARGIN = 1e-5
# (temperature, top_k, top_p, min_p)
SETTINGS = [(1.0, 0, 0.9, 0.0), (0.8, 0, 0.5, 0.0), (1.0, 64, 0.95, 0.0), (1.3, 0, 0.9, 0.02), (1.0, 0, 1.0, 0.05),
            (1.0, 0, 1e-6, 0.0)]
GREEDY_LIKE = 5   # the setting that must decode greedily
CASES = {   # geometry: (B, feature frames M -> T = M // 4 latent rows, speaker id, mfcc seed)
    "3d": (3, 120, 2, 4201),
    "6d": (2, 40, 1, 4202),
}


class WarpF:
    """torch.nn.functional with ``softmax`` replaced by the controlled warp (see the module docstring).  Records the
    size of every keep set, the two margins of every draw and whether the maximum logit was unique."""

    def __init__(self, temperature, top_k, top_p, min_p):
        self.t, self.k, self.p, self.m = float(temperature), int(top_k), float(top_p), float(min_p)
        self.kept, self.margin_p, self.margin_m, self.unique_max = [], [], [], []

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        assert logits.dim() == 2 and dim in (-1, 1)
        if self.t == 0:
            return TF.one_hot(torch.argmax(logits, dim), logits.shape[dim]).to(logits.dtype)
        keep = torch.ones_like(logits, dtype=torch.bool)
        if 0 < self.k < logits.shape[dim]:
            keep = logits >= torch.topk(logits, self.k, dim).values[..., -1:]
        s = logits / self.t
        e = torch.exp(s - logits.max(dim, keepdim=True).values / self.t).masked_fill(~keep, 0.0).numpy()   # fp32
        w = np.rint(e.astype(np.float64) * 2.0 ** 32)          # integers <= 2^32, exact in float64 like every sum below
        keep = keep.numpy().copy()
        mp = mm = np.inf
        rows_p, rows_m = [], []
        for b in range(logits.shape[0]):
            l = logits[b].numpy()
            self.unique_max.append(int((l == l.max()).sum()) == 1)
            if self.p < 1.0:
                _, cls = np.unique(l, return_inverse=True)           # tie classes, ascending; -0 and +0 are one class
                mass = np.bincount(cls, weights=w[b])
                above = (mass.sum() - np.cumsum(mass))[cls]          # mass of the strictly greater logits
                W = w[b].sum()
                P = float(np.float32(self.p)) * W
                keep[b] &= above < P
                rows_p.append(np.abs(above[above > 0] - P).min() / W if (above > 0).any() else np.inf)
            if self.m > 0.0:
                m = np.float32(self.m)
                keep[b] &= e[b] >= m
                rows_m.append(np.abs(e[b].astype(np.float64) - float(m)).min() / float(m))
        self.kept.append(keep.sum(1).astype(np.int32))
        self.margin_p.append(np.array(rows_p) if rows_p else np.full(logits.shape[0], mp))
        self.margin_m.append(np.array(rows_m) if rows_m else np.full(logits.shape[0], mm))
        return TF.softmax(s.masked_fill(~torch.from_numpy(keep), float("-inf")), dim)


def main():
    torch.set_num_threads(1)
    torch.set_grad_enabled(False)
    import_reference()
    import nets.smplx_body_pixel as ref_bp
    import nets.spg.gated_pixelcnn_v2 as ref_pix
    from trainer.config import load_JsonConfig

    tmp = tempfile.mkdtemp()
    a = types.SimpleNamespace(gpu="cpu", infer=True)
    out = {"settings": np.array(SETTINGS, dtype=np.float64), "seed": np.int64(SEED), "pose_stride": np.int64(POSE_STRIDE)}
    min_p, min_m = np.inf, np.inf
    for key, (B, M, spk, mseed) in CASES.items():
        six = key == "6d"
        vq = synth.body_vq_checkpoint_6d(0) if six else synth.body_vq_checkpoint(0)
        bp = synth.body_pixel_checkpoint_6d(0) if six else synth.body_pixel_checkpoint(0)
        vq_path = os.path.join(tmp, "vq_%s.pth" % key)
        torch.save({"generator": vq}, vq_path)
        cfg = load_JsonConfig("config/body_pixel.json")
        cfg.Data.pose.convert_to_6d = six
        cfg.Model.vq_path = vq_path
        g = ref_bp.TrainWrapper(a, cfg)
        g.load_state_dict(bp)
        mfcc = synth.synth_mfcc(1, M, seed=mseed)
        ref_bp.get_mfcc_ta = lambda *aa, **kk: mfcc[0].transpose(0, 1).numpy()   # (M, 64) like utils.py:177
        captured = []
        gen = g.generator.generate
        g.generator.generate = lambda *aa, **kk: captured.append(gen(*aa, **kk)) or captured[-1]
        out["mfcc_%s" % key] = mfcc.numpy()
        out["label_%s" % key] = np.int64(spk)
        out["fp_%s" % key] = np.array(list(synth.fingerprint(bp).values()))
        out["fp_vq_%s" % key] = np.array(list(synth.fingerprint(vq).values()))

        def run(warp, seed):
            ref_pix.F = warp
            captured.clear()
            torch.manual_seed(seed)
            pred = g.infer_on_audio("synthetic.wav", id=torch.tensor([spk]), fps=30, B=B)    # (B, 4T, C)
            ref_pix.F = TF
            return captured[0], np.asarray(pred, dtype=np.float32)

        seeds = []
        for i, (t, k, p, m) in enumerate(SETTINGS):
            seed = SEED + i
            while True:
                warp = WarpF(t, k, p, m)
                codes, pred = run(warp, seed)
                mp, mm = float(np.min(warp.margin_p)), float(np.min(warp.margin_m))
                if min(mp, mm) >= MIN_MARGIN:
                    break
                print("nucleus", key, (t, k, p, m), "seed", seed, "margins %.3g %.3g: next seed" % (mp, mm), flush=True)
                seed += 100
            seeds.append(seed)
            T = codes.shape[1]
            kept = np.stack(warp.kept, 0).reshape(T, 2, B).transpose(2, 0, 1)          # one softmax per (row, column)
            min_p, min_m = min(min_p, mp), min(min_m, mm)
            if i == GREEDY_LIKE:
                assert all(warp.unique_max), "a draw has tied maximum logits: choose another seed"
                greedy, _ = run(WarpF(0.0, 0, 1.0, 0.0), seed)
                assert torch.equal(codes, greedy), "top_p -> 0 must decode greedily"
                assert (kept == 1).all()
            out["codes_%s_%d" % (key, i)] = codes.numpy()
            out["kept_%s_%d" % (key, i)] = np.ascontiguousarray(kept)
            out["poses_%s_%d" % (key, i)] = np.ascontiguousarray(pred[:, ::POSE_STRIDE])
            print("nucleus", key, (t, k, p, m), codes[0, :3].tolist(), "kept", int(kept.min()), int(kept.max()),
                  "margins %.3g %.3g" % (mp, mm), flush=True)
        out["seeds_%s" % key] = np.array(seeds, dtype=np.int64)
    out["min_margin_top_p"] = np.float64(min_p)
    out["min_margin_min_p"] = np.float64(min_m)
    print("smallest margins: top_p %.3g, min_p %.3g" % (min_p, min_m), flush=True)
    assert min(min_p, min_m) >= MIN_MARGIN
    np.savez_compressed(os.path.join(HERE, "sampling_p.npz"), **out)


if __name__ == "__main__":
    main()
