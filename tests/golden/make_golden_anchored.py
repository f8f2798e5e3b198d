"""Generate tests/golden/anchored.npz: codes, per-draw log p and poses of the UNMODIFIED reference's
s2g_body_pixel.infer_on_audio (nets/smplx_body_pixel.py:232-289) with chosen draws pinned to given codes (anchored
sampling, ts_body_sample_anchored in include/talkshow_b200.h).  Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_anchored.py

The module's ``F`` is swapped for a proxy.  The reference calls ``F.softmax`` once per (row, column) of the generate loop,
in order (gated_pixelcnn_v2.py:167-176), so the proxy knows which draw each call is for by counting.  For a pinned sample
it returns a one-hot at the anchor: ``torch.multinomial`` still draws its [B, 2048] exponentials, so the RNG stream stays
the reference's, and it returns the anchor.  Unpinned samples get the warp of the setting (make_golden_nucleus.WarpF, the
controls of ts_pixelcnn_sample_ctl).  The proxy also records the reference's ``log_softmax`` of every call's logits, so
the log p of every draw, pinned or sampled, is read at the code the loop kept.

Patterns (per setting): none pinned, a pinned prefix, a free window inside pinned rows, the body column only, the hand
column only, a scattered 30 % and everything.  The anchors are the codes of the setting's unanchored run, except for the
scattered pattern, which pins uniform random codes (some of them far from what the prior would draw).  The top-p setting
reuses the rule of make_golden_nucleus.py: a run whose smallest keep-set margin over the SAMPLED draws is below MIN_MARGIN
is repeated under the next seed (seed + 100, ...).  Running the script again reproduces the file byte for byte (fixed
seeds, CPU, one thread).
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

from make_golden_nucleus import WarpF  # noqa: E402
from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

SEED = 5100
POSE_STRIDE = 10   # poses are kept for every 10th frame (the codes, which determine them, are kept whole)
MIN_MARGIN = 1e-5
SETTINGS = [(1.0, 0, 1.0), (0.8, 64, 1.0), (1.0, 0, 0.9)]     # (temperature, top_k, top_p): default, tempered top-k, top-p
PATTERNS = ["none", "prefix", "window", "body", "hand", "scattered", "all"]
CASES = {   # geometry: (B, feature frames M -> T = M // 4 latent rows, speaker id, mfcc seed)
    "3d": (3, 120, 2, 5201),
    "6d": (2, 40, 1, 5202),
}


def pattern(name, B, T, free_codes, seed):
    """anchors [B,T,2] int64 of one pattern (-1 = sampled)"""
    a = np.full((B, T, 2), -1, dtype=np.int64)
    if name == "prefix":
        a[:, :T // 3] = free_codes[:, :T // 3]
    elif name == "window":
        a[:] = free_codes
        a[:, T // 3: 2 * T // 3] = -1
    elif name == "body":
        a[..., 0] = free_codes[..., 0]
    elif name == "hand":
        a[..., 1] = free_codes[..., 1]
    elif name == "scattered":
        rng = np.random.RandomState(seed)
        codes = rng.randint(0, 2048, size=(B, T, 2))
        a = np.where(rng.rand(B, T, 2) < 0.3, codes, -1).astype(np.int64)
    elif name == "all":
        a[:] = free_codes
    return a


class AnchoredF:
    """torch.nn.functional whose ``softmax`` pins the draws ``anchors`` [B,T,2] pins (one-hot at the anchor) and warps the
    others (WarpF); records log_softmax of every call's logits."""

    def __init__(self, anchors, warp):
        self.anchors, self.warp, self.n, self.logsm = anchors, warp, 0, []

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        i, j = divmod(self.n, 2)
        self.n += 1
        self.logsm.append(TF.log_softmax(logits, dim).numpy())
        p = self.warp.softmax(logits, dim)
        pin = self.anchors[:, i, j] >= 0
        if self.warp.p < 1.0:   # a pinned draw has no keep set: its margin does not count
            self.warp.margin_p[-1] = np.where(pin, np.inf, self.warp.margin_p[-1])
        if pin.any():
            one = TF.one_hot(torch.from_numpy(np.maximum(self.anchors[:, i, j], 0)), logits.shape[dim]).to(p.dtype)
            p = torch.where(torch.from_numpy(pin)[:, None], one, p)
        return p


def main():
    torch.set_num_threads(1)
    torch.set_grad_enabled(False)
    import_reference()
    import nets.smplx_body_pixel as ref_bp
    import nets.spg.gated_pixelcnn_v2 as ref_pix
    from trainer.config import load_JsonConfig

    tmp = tempfile.mkdtemp()
    a = types.SimpleNamespace(gpu="cpu", infer=True)
    out = {}
    for key, (B, M, spk, mseed) in CASES.items():
        six = key == "6d"
        T = M // 4
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

        def run(anchors, setting, seed):
            proxy = AnchoredF(anchors, WarpF(setting[0], setting[1], setting[2], 0.0))
            ref_pix.F = proxy
            captured.clear()
            torch.manual_seed(seed)
            pred = g.infer_on_audio("synthetic.wav", id=torch.tensor([spk]), fps=30, B=B)    # (B, 4T, C)
            ref_pix.F = TF
            assert proxy.n == 2 * T
            codes = captured[0].numpy()
            logsm = np.stack(proxy.logsm, 0).reshape(T, 2, B, -1)                            # one call per (row, column)
            logp = np.take_along_axis(logsm, codes.transpose(1, 2, 0)[..., None], -1)[..., 0].transpose(2, 0, 1)
            margin = float(np.min(proxy.warp.margin_p)) if setting[2] < 1.0 else np.inf
            return codes, np.ascontiguousarray(logp, dtype=np.float32), np.asarray(pred, dtype=np.float32), margin

        names, settings, anchors_all, seeds, codes_all, logp_all, poses_all = [], [], [], [], [], [], []
        for si, setting in enumerate(SETTINGS):
            free = None
            for pi, name in enumerate(PATTERNS):
                seed = SEED + 10 * si + pi
                anchors = pattern(name, B, T, free, seed) if free is not None else np.full((B, T, 2), -1, dtype=np.int64)
                while True:
                    codes, logp, pred, margin = run(anchors, setting, seed)
                    if margin >= MIN_MARGIN:
                        break
                    print("anchored", key, setting, name, "seed", seed, "margin %.3g: next seed" % margin, flush=True)
                    seed += 100
                pin = anchors >= 0
                assert (codes[pin] == anchors[pin]).all()
                if free is None:
                    free = codes
                names.append("%s/%s" % ("t%g-k%d-p%g" % setting, name))
                settings.append(setting)
                anchors_all.append(anchors)
                seeds.append(seed)
                codes_all.append(codes)
                logp_all.append(logp)
                poses_all.append(pred[:, ::POSE_STRIDE])
                print("anchored", key, names[-1], "seed", seed, "pinned %d / %d" % (pin.sum(), pin.size),
                      codes[0, :3].tolist(), flush=True)
        out[key + "_mfcc"] = mfcc.repeat(B, 1, 1).numpy()
        out[key + "_label"] = np.full(B, spk, dtype=np.int64)
        out[key + "_pose_stride"] = np.int64(POSE_STRIDE)
        out[key + "_cases"] = np.array(names)
        out[key + "_setting"] = np.array(settings, dtype=np.float64)
        out[key + "_anchors"] = np.stack(anchors_all)
        out[key + "_seed"] = np.array(seeds, dtype=np.int64)
        out[key + "_codes"] = np.stack(codes_all)
        out[key + "_logp"] = np.stack(logp_all)
        out[key + "_poses"] = np.ascontiguousarray(np.stack(poses_all))
        out[key + "_fp"] = np.array(list(synth.fingerprint(bp).values()))
        out[key + "_fp_vq"] = np.array(list(synth.fingerprint(vq).values()))
    np.savez_compressed(os.path.join(HERE, "anchored.npz"), **out)


if __name__ == "__main__":
    main()
