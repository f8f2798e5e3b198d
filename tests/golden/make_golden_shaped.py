"""Generate tests/golden/shaped.npz: codes and poses of the UNMODIFIED reference's s2g_body_pixel.infer_on_audio
(nets/smplx_body_pixel.py:232-289) and GatedPixelCNN.generate (nets/spg/gated_pixelcnn_v2.py:152-177) for one batch
whose clips draw under logit shaping (repetition penalty and code bias, ts_pixelcnn_sample_shaped).  Run on a host with a
reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_shaped.py

The recipe is that of make_golden_clip_ctl.py.  The generator's ``forward`` is wrapped to record the code grid x it is
given: every forward sees every earlier draw, the pre_latents prefix included.  The module's ``F`` is swapped for a proxy
whose ``softmax``, for batch row b at step (i, j), shapes the raw logits and then applies the warp of clip b's controls
(make_golden_nucleus.WarpF; a greedy row is the one-hot of the argmax of the shaped logits):
  - penalty: every code in x[b, max(0, i - W):i, j] (once) gets l / theta where l > 0, l * theta otherwise (fp32);
  - bias: l + bias[b, j] (fp32).
A code whose shaped logit is -inf has probability 0 and is not counted in the keep set.  Everything else (the loop, the
multinomial draw under the seed, the VQ decoders) is the reference's own code.  Case "3d" runs infer_on_audio; case
"pre" runs GatedPixelCNN.generate with a pre_latents prefix that the windows reach into; case "6d" runs infer_on_audio on
the convert_to_6d geometry.

Draw-margin rule (as in sampling_p.npz): a run whose smallest nucleus or min-p margin is below MIN_MARGIN is repeated
under the next seed (seed + 100, ...).  The greedy rows must have a unique maximum shaped logit at every draw (asserted).
Running the script again reproduces the file byte for byte (fixed seeds, CPU, one thread).
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

SEED = 6100
POSE_STRIDE = 5
NCODE = 2048
# (temperature, top_k, top_p, min_p, repetition_penalty, repetition_window, bias kind) of clip b
SETTINGS = [
    (1.0, 0, 1.0, 0.0, 1.0, 8, "none"),          # the default draw
    (1.0, 0, 1.0, 0.0, 1.5, 1, "none"),
    (1.0, 0, 1.0, 0.0, 1.5, 8, "none"),
    (1.0, 0, 1.0, 0.0, 3.0, 100000, "none"),     # the whole history
    (0.0, 0, 1.0, 0.0, 2.0, 4, "none"),          # greedy + penalty
    (0.0, 0, 1.0, 0.0, 2.0, 4, "ban"),           # greedy + penalty + a ban list
    (1.0, 0, 1.0, 0.0, 1.0, 8, "even_body"),     # even body codes banned
    (1.0, 0, 1.0, 0.0, 1.0, 8, "hand16"),        # the hand column limited to 16 codes
    (1.0, 0, 1.0, 0.0, 1.0, 8, "normal"),        # a random N(0, 1) bias
    (0.8, 0, 0.9, 0.0, 1.3, 8, "none"),
    (1.0, 0, 1.0, 0.05, 1.3, 8, "none"),
    (1.0, 0, 1.0, 0.0, 1.0, 8, "one"),           # all but one code banned
]
GREEDY_ROWS = [b for b, s in enumerate(SETTINGS) if s[0] == 0.0]
CASES = {   # case: (geometry, feature frames M -> T = M // 4 latent rows, speaker id, mfcc seed, prefix rows)
    "3d": ("3d", 120, 2, 6201, 0),
    "pre": ("3d", 40, 1, 6203, 12),
    "6d": ("6d", 40, 1, 6202, 0),
}


def make_bias(seed):
    """[B,2,2048] float32 bias rows of SETTINGS (zeros where the kind is "none")"""
    rng = np.random.RandomState(seed)
    bias = np.zeros((len(SETTINGS), 2, NCODE), np.float32)
    for b, s in enumerate(SETTINGS):
        kind = s[6]
        if kind == "ban":
            for c in range(2):
                bias[b, c, rng.choice(NCODE, 512, replace=False)] = -np.inf
        elif kind == "even_body":
            bias[b, 0, 0::2] = -np.inf
        elif kind == "hand16":
            bias[b, 1] = -np.inf
            bias[b, 1, rng.choice(NCODE, 16, replace=False)] = 0.0
        elif kind == "normal":
            bias[b] = rng.standard_normal((2, NCODE)).astype(np.float32)
        elif kind == "one":
            bias[b] = -np.inf
            bias[b, :, rng.randint(NCODE)] = 0.0
    return bias


class ShapedF:
    """torch.nn.functional with ``softmax`` replaced by, for each batch row b, the shaping of clip b followed by the warp
    of its controls.  ``grid`` holds the code tensor the last forward saw; ``h0`` is the first row drawn."""

    def __init__(self, bias, h0):
        self.warps = [WarpF(*s[:4]) for s in SETTINGS]
        self.bias = torch.from_numpy(bias)
        self.grid, self.h0, self.step = [None], h0, 0
        self.kept = [[] for _ in SETTINGS]
        self.unique_max = [[] for _ in SETTINGS]

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        assert logits.dim() == 2 and dim in (-1, 1) and logits.shape[0] == len(SETTINGS)
        i, j = self.h0 + self.step // 2, self.step % 2
        self.step += 1
        x = self.grid[0]
        rows = []
        for b, (t, k, p, m, theta, W, _) in enumerate(SETTINGS):
            l = logits[b].clone()
            hist = torch.unique(x[b, max(0, i - W):i, j])
            if theta != 1.0 and hist.numel():
                v = l[hist]
                l[hist] = torch.where(v > 0, v / np.float32(theta), v * np.float32(theta))
            l = l + self.bias[b, j]
            self.unique_max[b].append(int((l == l.max()).sum()) == 1)
            rows.append(self.warps[b].softmax(l[None], dim))
            # WarpF counts the -inf codes that top-k leaves in (top_p / min_p drop them): they have probability 0 and are
            # not in the keep set
            ninf = int((l == float("-inf")).sum())
            nfin = NCODE - ninf
            if t > 0:
                left = ninf if (p >= 1.0 and m <= 0.0 and (not 0 < k < NCODE or nfin < k)) else 0
                self.kept[b].append(int(self.warps[b].kept[-1][0]) - left)
            else:
                self.kept[b].append(1)
        return torch.cat(rows, 0)

    def margins(self):
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
    out = {"settings": np.array([s[:6] for s in SETTINGS], dtype=np.float64), "pose_stride": np.int64(POSE_STRIDE)}
    min_p, min_m = np.inf, np.inf
    for ci, (case, (geo, M, spk, mseed, T0)) in enumerate(CASES.items()):
        six = geo == "6d"
        vq = synth.body_vq_checkpoint_6d(0) if six else synth.body_vq_checkpoint(0)
        bp = synth.body_pixel_checkpoint_6d(0) if six else synth.body_pixel_checkpoint(0)
        vq_path = os.path.join(tmp, "vq_%s.pth" % case)
        torch.save({"generator": vq}, vq_path)
        cfg = load_JsonConfig("config/body_pixel.json")
        cfg.Data.pose.convert_to_6d = six
        cfg.Model.vq_path = vq_path
        g = ref_bp.TrainWrapper(a, cfg)
        g.load_state_dict(bp)
        mfcc = synth.synth_mfcc(1, M, seed=mseed)
        bias = make_bias(mseed)
        out["mfcc_%s" % case] = mfcc.numpy()
        out["label_%s" % case] = np.int64(spk)
        out["bias_%s" % case] = bias
        out["fp_%s" % case] = np.array(list(synth.fingerprint(bp).values()))
        out["fp_vq_%s" % case] = np.array(list(synth.fingerprint(vq).values()))
        fwd = g.generator.forward
        captured = []
        gen = g.generator.generate
        g.generator.generate = lambda *aa, **kk: captured.append(gen(*aa, **kk)) or captured[-1]
        if T0:
            rng = np.random.RandomState(mseed + 1)
            pre = rng.randint(0, NCODE, size=(B, T0, 2)).astype(np.int64)
            # repeated codes in the prefix's last rows, so the windows find them there
            pre[:, -4:, :] = pre[:, -5:-4, :]
            mfcc_pre = synth.synth_mfcc(1, 4 * T0, seed=mseed + 2)
            out["pre_%s" % case] = pre
            out["mfcc_pre_%s" % case] = mfcc_pre.numpy()
            g.generator.eval()           # as s2g_body_pixel.generate (:306-316) before it runs the audio encoder
            g.audioencoder.eval()
            aud = g.audioencoder(mfcc.repeat(B, 1, 1), frame_num=0).unsqueeze(-1).repeat(1, 1, 1, 2)
            aud_pre = g.audioencoder(mfcc_pre.repeat(B, 1, 1), frame_num=0).unsqueeze(-1).repeat(1, 1, 1, 2)
        else:
            ref_bp.get_mfcc_ta = lambda *aa, **kk: mfcc[0].transpose(0, 1).numpy()   # (M, 64) like utils.py:177

        seed = SEED + ci
        while True:
            warp = ShapedF(bias, T0)

            def record(x, *aa, **kk):
                warp.grid[0] = x
                return fwd(x, *aa, **kk)

            g.generator.forward = record
            ref_pix.F = warp
            captured.clear()
            torch.manual_seed(seed)
            if T0:
                codes = g.generator.generate(torch.full((B,), spk), shape=[aud.shape[2], 2], batch_size=B, aud_feat=aud,
                                             pre_latents=torch.from_numpy(pre), pre_audio=aud_pre)
                pred = None
            else:
                pred = np.asarray(g.infer_on_audio("synthetic.wav", id=torch.tensor([spk]), fps=30, B=B), dtype=np.float32)
                codes = captured[0]
            ref_pix.F = TF
            g.generator.forward = fwd
            mp, mm = warp.margins()
            if min(mp, mm) >= MIN_MARGIN:
                break
            print("shaped", case, "seed", seed, "margins %.3g %.3g: next seed" % (mp, mm), flush=True)
            seed += 100
        for b in GREEDY_ROWS:
            assert all(warp.unique_max[b]), "clip %d: a draw has tied maximum shaped logits: choose another seed" % b
        T = codes.shape[1]
        kept = np.array(warp.kept, dtype=np.int32).reshape(B, T, 2)
        assert (kept >= 1).all()
        min_p, min_m = min(min_p, mp), min(min_m, mm)
        out["seed_%s" % case] = np.int64(seed)
        out["codes_%s" % case] = codes.numpy()
        out["kept_%s" % case] = np.ascontiguousarray(kept)
        if pred is not None:
            out["poses_%s" % case] = np.ascontiguousarray(pred[:, ::POSE_STRIDE])
        print("shaped", case, "seed", seed, codes[:, 0, 0].tolist(), "kept", kept.min(axis=(1, 2)).tolist(),
              "margins %.3g %.3g" % (mp, mm), flush=True)
    out["min_margin_top_p"] = np.float64(min_p)
    out["min_margin_min_p"] = np.float64(min_m)
    assert min(min_p, min_m) >= MIN_MARGIN
    np.savez_compressed(os.path.join(HERE, "shaped.npz"), **out)


if __name__ == "__main__":
    main()
