"""Generate tests/golden/clip_ctl.npz: codes and poses of the UNMODIFIED reference's s2g_body_pixel.infer_on_audio
(nets/smplx_body_pixel.py:232-289) for ONE batch whose clips draw under different sampling controls (per-clip controls,
ts_pixelcnn_sample_clips).  Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_clip_ctl.py

The recipe is that of make_golden_sampling.py and make_golden_nucleus.py: the module's ``F`` is swapped for a proxy whose
``softmax`` applies, to batch row b, the warp of clip b's setting (make_golden_nucleus.WarpF, one row at a time; a
greedy row is the one-hot of its argmax).  The batch holds every setting of sampling.npz and sampling_p.npz plus a default
clip and a second greedy clip whose top_k / top_p / min_p must be ignored, in an order that puts greedy clips between
sampled ones.  Everything else (the loop, the multinomial draw under the seed, the VQ decoders) is the reference's own
code; every clip sees the same audio and the same speaker, so clips differ only by their noise and their setting.

Draw-margin rule (as in sampling_p.npz): a run whose smallest nucleus or min-p margin, over the clips with those
truncations on, is below MIN_MARGIN is repeated under the next seed (seed + 100, ...), so no keep set of the fixture is
ambiguous between the CPU's exp and the GPU's expf.  The greedy rows and the top_p = 1e-6 row must have a unique maximum
logit at every draw (asserted), so their first-index argmax is unambiguous.  Running the script again reproduces the file
byte for byte (fixed seeds, CPU, one thread).
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

from make_golden_nucleus import MIN_MARGIN, WarpF  # noqa: E402
from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

SEED = 5100
POSE_STRIDE = 5
# (temperature, top_k, top_p, min_p) of clip b: sampling.npz's settings, sampling_p.npz's settings, the default draw and a
# greedy clip with truncations that greedy decoding ignores
SETTINGS = [(0.7, 0, 1.0, 0.0), (1.0, 0, 0.9, 0.0), (0.0, 0, 1.0, 0.0), (1.3, 0, 1.0, 0.0), (0.8, 0, 0.5, 0.0),
            (1.0, 5, 1.0, 0.0), (1.0, 64, 0.95, 0.0), (0.0, 5, 0.5, 0.1), (0.8, 64, 1.0, 0.0), (1.3, 0, 0.9, 0.02),
            (1.0, 0, 1.0, 0.0), (1.0, 0, 1.0, 0.05), (1.0, 0, 1e-6, 0.0)]
ARGMAX_ROWS = [b for b, (t, k, p, m) in enumerate(SETTINGS) if t == 0.0 or p == 1e-6]   # must have a unique max
CASES = {   # geometry: (feature frames M -> T = M // 4 latent rows, speaker id, mfcc seed)
    "3d": (120, 2, 5201),
    "6d": (40, 1, 5202),
}


class ClipWarpF:
    """torch.nn.functional with ``softmax`` replaced by, for each batch row b, the warp of SETTINGS[b] (WarpF on that row
    alone).  Records every row's keep-set size and margins and whether its maximum logit was unique."""

    def __init__(self, settings):
        self.warps = [WarpF(*s) for s in settings]
        self.unique_max = [[] for _ in settings]

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        assert logits.dim() == 2 and dim in (-1, 1) and logits.shape[0] == len(self.warps)
        for b in range(logits.shape[0]):
            self.unique_max[b].append(int((logits[b] == logits[b].max()).sum()) == 1)
        return torch.cat([w.softmax(logits[b:b + 1], dim) for b, w in enumerate(self.warps)], 0)

    def margins(self):
        """smallest nucleus and min-p margins over the clips with that truncation on (inf when none)"""
        mp = [float(np.min(w.margin_p)) for w in self.warps if w.t > 0 and w.p < 1.0]
        mm = [float(np.min(w.margin_m)) for w in self.warps if w.t > 0 and w.m > 0.0]
        return min(mp, default=np.inf), min(mm, default=np.inf)


def main():
    torch.set_num_threads(1)
    torch.set_grad_enabled(False)
    import_reference()
    import nets.smplx_body_pixel as ref_bp
    import nets.spg.gated_pixelcnn_v2 as ref_pix
    from trainer.config import load_JsonConfig

    tmp = tempfile.mkdtemp()
    a = types.SimpleNamespace(gpu="cpu", infer=True)
    B = len(SETTINGS)
    out = {"settings": np.array(SETTINGS, dtype=np.float64), "pose_stride": np.int64(POSE_STRIDE)}
    min_p, min_m = np.inf, np.inf
    for key, (M, spk, mseed) in CASES.items():
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

        seed = SEED + (1 if six else 0)
        while True:
            warp = ClipWarpF(SETTINGS)
            ref_pix.F = warp
            captured.clear()
            torch.manual_seed(seed)
            pred = np.asarray(g.infer_on_audio("synthetic.wav", id=torch.tensor([spk]), fps=30, B=B), dtype=np.float32)
            ref_pix.F = TF
            codes = captured[0]
            mp, mm = warp.margins()
            if min(mp, mm) >= MIN_MARGIN:
                break
            print("clip_ctl", key, "seed", seed, "margins %.3g %.3g: next seed" % (mp, mm), flush=True)
            seed += 100
        for b in ARGMAX_ROWS:
            assert all(warp.unique_max[b]), "clip %d: a draw has tied maximum logits: choose another seed" % b
        T = codes.shape[1]
        # one softmax per (row, column); a greedy draw keeps one code (include/talkshow_b200.h)
        kept = np.stack([np.concatenate(w.kept) if w.t > 0 else np.ones(2 * T, np.int32) for w in warp.warps], 0)
        kept = kept.reshape(B, T, 2)
        min_p, min_m = min(min_p, mp), min(min_m, mm)
        out["seed_%s" % key] = np.int64(seed)
        out["codes_%s" % key] = codes.numpy()
        out["kept_%s" % key] = np.ascontiguousarray(kept)
        out["poses_%s" % key] = np.ascontiguousarray(pred[:, ::POSE_STRIDE])
        print("clip_ctl", key, "seed", seed, codes[:, 0, 0].tolist(), "kept", kept.min(axis=(1, 2)).tolist(),
              "margins %.3g %.3g" % (mp, mm), flush=True)
    out["min_margin_top_p"] = np.float64(min_p)
    out["min_margin_min_p"] = np.float64(min_m)
    assert min(min_p, min_m) >= MIN_MARGIN
    np.savez_compressed(os.path.join(HERE, "clip_ctl.npz"), **out)


if __name__ == "__main__":
    main()
