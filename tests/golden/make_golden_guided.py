"""Generate tests/golden/guided.npz: codes and keep-set sizes of the UNMODIFIED reference's GatedPixelCNN.generate
(nets/spg/gated_pixelcnn_v2.py:152-177) run on 2P interleaved rows under guided sampling (ts_pixelcnn_sample_guided).
Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_guided.py

Row 2p is clip p and row 2p + 1 its negative conditioning: its own audio features (encoded by the reference's audio
encoder) and its own label, or, in case "style", its own speaker weights through make_golden_style.BlendEmbedding (the
clip's row one-hot, the negative's the uniform blend).  The recipe is that of make_golden_shaped.py.  The generator's
``forward`` is wrapped to record the code grid x it is given.  The module's ``F`` is swapped for a proxy whose
``softmax``, for rows (2p, 2p + 1) at step (i, j):
  - forms g = l_c + (w_p - 1)(l_c - l_u) from the two rows' logits, three separately rounded fp32 operations (numpy);
  - applies pair p's shaping (penalty over x[2p, max(0, i - W):i, j], then its bias row) and the warp of its controls
    (make_golden_nucleus.WarpF; a greedy pair is the one-hot of the argmax);
  - returns those probabilities for both rows, as a tensor whose ``multinomial`` draws the even rows only and gives each
    odd row its even row's code.
So the reference's own loop feeds both branches the guided code, and the draw consumes the Exp(1) noise of a P-row batch
under the seed: the pair noise is ``oracle_sampling.reference_noise(seed, 2T, P)``.  Everything else (the loop, the
networks, the multinomial) is the reference's own code.

The "silence" negative is flat features (every frame the same zero vector), standing in for a silent clip; the fixture
stores the features, so the tests feed exactly these.  Cases: "3d" (negatives: flat audio, another speaker, both), "style"
(negative: the uniform blend of the four speakers), "pre" (a pre_latents prefix fed to both rows, each branch with its own
prefix audio), "6d" (the convert_to_6d geometry).

Draw-margin rule (as in sampling_p.npz): a run whose smallest nucleus or min-p margin is below MIN_MARGIN is repeated
under the next seed (seed + 100, ...).  The greedy pairs must have a unique maximum guided logit at every draw (asserted).
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
from make_golden_style import BlendEmbedding  # noqa: E402
from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

SEED = 7100
NCODE = 2048
NCLS = 4
# (temperature, top_k, top_p, min_p, repetition_penalty, repetition_window, ban list, guidance w, negative) of pair p;
# negative: "silence" (flat audio, same speaker), "speaker" (same audio, speaker + 1), "both"
SETTINGS = [
    (1.0, 0, 1.0, 0.0, 1.0, 8, 0, 1.0, "silence"),
    (1.0, 0, 1.0, 0.0, 1.0, 8, 0, 2.0, "silence"),
    (1.0, 0, 1.0, 0.0, 1.0, 8, 0, 3.0, "speaker"),
    (1.0, 0, 1.0, 0.0, 1.0, 8, 0, 0.5, "both"),
    (0.8, 0, 0.9, 0.0, 1.0, 8, 0, 1.5, "speaker"),    # tempered nucleus
    (0.0, 0, 1.0, 0.0, 2.0, 4, 0, 2.0, "silence"),    # greedy + penalty
    (1.0, 0, 1.0, 0.0, 1.0, 8, 1, 3.0, "both"),       # a ban list
    (1.0, 0, 1.0, 0.05, 1.0, 8, 0, 1.5, "both"),      # min-p
    (1.0, 64, 1.0, 0.0, 1.5, 8, 0, 2.0, "speaker"),   # top-k + penalty
]
GREEDY = [p for p, s in enumerate(SETTINGS) if s[0] == 0.0]
CASES = {   # case: (geometry, feature frames M -> T = M // 4 latent rows, speaker id, mfcc seed, prefix rows)
    "3d": ("3d", 120, 1, 7201, 0),
    "style": ("3d", 40, 2, 7202, 0),
    "pre": ("3d", 40, 0, 7203, 12),
    "6d": ("6d", 40, 3, 7204, 0),
}


def make_bias(seed):
    """[P,2,2048] float32 bias rows: 512 banned codes per column for the pairs with a ban list, zeros elsewhere"""
    rng = np.random.RandomState(seed)
    bias = np.zeros((len(SETTINGS), 2, NCODE), np.float32)
    for p, s in enumerate(SETTINGS):
        if s[6]:
            for c in range(2):
                bias[p, c, rng.choice(NCODE, 512, replace=False)] = -np.inf
    return bias


def guided(lc, lu, w):
    """g = lc + (w - 1)(lc - lu), each operation rounded to fp32"""
    s = np.float32(np.float32(w) - np.float32(1.0))
    return torch.from_numpy(np.float32(lc + np.float32(s * np.float32(lc - lu))))


class PairProbs(torch.Tensor):
    """probabilities of 2P rows whose multinomial draws the even rows and repeats each code for the odd row"""

    def multinomial(self, n, *a, **k):
        even = self.as_subclass(torch.Tensor)[0::2]
        return torch.Tensor.multinomial(even, n, *a, **k).repeat_interleave(2, 0)


class GuidedF:
    """torch.nn.functional with ``softmax`` replaced by the guided draw of each pair (see the module docstring)."""

    def __init__(self, bias, h0):
        self.warps = [WarpF(*s[:4]) for s in SETTINGS]
        self.bias = torch.from_numpy(bias)
        self.grid, self.h0, self.step = [None], h0, 0
        self.kept = [[] for _ in SETTINGS]
        self.unique_max = [[] for _ in SETTINGS]

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        assert logits.dim() == 2 and dim in (-1, 1) and logits.shape[0] == 2 * len(SETTINGS)
        i, j = self.h0 + self.step // 2, self.step % 2
        self.step += 1
        x = self.grid[0]
        rows = []
        for p, (t, k, tp, mp, theta, W, _, w, _) in enumerate(SETTINGS):
            assert torch.equal(x[2 * p, :i], x[2 * p + 1, :i])      # both branches were fed the same codes
            l = guided(logits[2 * p].numpy(), logits[2 * p + 1].numpy(), w)
            hist = torch.unique(x[2 * p, max(0, i - W):i, j])
            if theta != 1.0 and hist.numel():
                v = l[hist]
                l[hist] = torch.where(v > 0, v / np.float32(theta), v * np.float32(theta))
            l = l + self.bias[p, j]
            self.unique_max[p].append(int((l == l.max()).sum()) == 1)
            r = self.warps[p].softmax(l[None], dim)
            rows += [r, r]
            ninf = int((l == float("-inf")).sum())
            if t > 0:   # WarpF counts the -inf codes top-k leaves in; they have probability 0 and are not kept
                left = ninf if (tp >= 1.0 and mp <= 0.0 and (not 0 < k < NCODE or NCODE - ninf < k)) else 0
                self.kept[p].append(int(self.warps[p].kept[-1][0]) - left)
            else:
                self.kept[p].append(1)
        return torch.cat(rows, 0).as_subclass(PairProbs)

    def margins(self):
        mp = [float(np.min(w.margin_p)) for w in self.warps if w.t > 0 and w.p < 1.0]
        mm = [float(np.min(w.margin_m)) for w in self.warps if w.t > 0 and w.m > 0.0]
        return min(mp, default=np.inf), min(mm, default=np.inf)


def branches(clip, neg, kinds):
    """rows 2p = clip[p], 2p + 1 = neg[p] where pair p's negative involves that field, else clip[p]"""
    out = []
    for p, kind in enumerate(kinds):
        out += [clip[p], neg[p] if kind else clip[p]]
    return torch.stack(out, 0)


def main():
    torch.set_num_threads(1)
    torch.set_grad_enabled(False)
    import_reference()
    import nets.smplx_body_pixel as ref_bp
    import nets.spg.gated_pixelcnn_v2 as ref_pix
    from trainer.config import load_JsonConfig

    tmp = tempfile.mkdtemp()
    a = types.SimpleNamespace(gpu="cpu", infer=True)
    P = len(SETTINGS)
    out = {"settings": np.array([s[:6] + (s[7],) for s in SETTINGS], dtype=np.float64),
           "negative": np.array([s[8] for s in SETTINGS])}
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
        g.generator.eval()
        g.audioencoder.eval()
        styled = case == "style"
        # the negative's audio and label per pair; the style case's negative is the uniform blend only
        neg_audio = [not styled and s[8] in ("silence", "both") for s in SETTINGS]
        neg_label = [not styled and s[8] in ("speaker", "both") for s in SETTINGS]
        mfcc = synth.synth_mfcc(1, M, seed=mseed)
        flat = torch.zeros(1, 64, M)
        mfcc2 = branches(mfcc.repeat(P, 1, 1), flat.repeat(P, 1, 1), neg_audio)
        labels = torch.full((P,), spk)
        label2 = branches(labels, (labels + 1) % NCLS, neg_label)
        bias = make_bias(mseed)
        out["mfcc_%s" % case] = mfcc.numpy()
        out["mfcc_neg_%s" % case] = flat.numpy()
        out["label_%s" % case] = np.int64(spk)
        out["bias_%s" % case] = bias
        out["fp_%s" % case] = np.array(list(synth.fingerprint(bp).values()))
        aud = g.audioencoder(mfcc2, frame_num=0).unsqueeze(-1).repeat(1, 1, 1, 2)
        pre = aud_pre = None
        if T0:
            rng = np.random.RandomState(mseed + 1)
            pre = rng.randint(0, NCODE, size=(P, T0, 2)).astype(np.int64)
            pre[:, -4:, :] = pre[:, -5:-4, :]                       # repeats the penalty windows reach
            mfcc_pre = synth.synth_mfcc(1, 4 * T0, seed=mseed + 2)
            out["pre_%s" % case] = pre
            out["mfcc_pre_%s" % case] = mfcc_pre.numpy()
            mpre2 = branches(mfcc_pre.repeat(P, 1, 1), torch.zeros(P, 64, 4 * T0), neg_audio)
            aud_pre = g.audioencoder(mpre2, frame_num=0).unsqueeze(-1).repeat(1, 1, 1, 2)
            pre = torch.from_numpy(pre).repeat_interleave(2, 0)
        cond = label2
        embs = []
        if styled:   # every layer's class term from per-row weights: one-hot of the clip's speaker, uniform for the negative
            w = torch.zeros(2 * P, NCLS)
            w[0::2, spk] = 1.0
            w[1::2] = 1.0 / NCLS
            cond = w
            for layer in g.generator.layers:
                embs.append(layer.class_cond_embedding)
                layer.class_cond_embedding = BlendEmbedding(layer.class_cond_embedding)
        fwd = g.generator.forward
        seed = SEED + ci
        while True:
            warp = GuidedF(bias, T0)

            def record(x, *aa, **kk):
                warp.grid[0] = x
                return fwd(x, *aa, **kk)

            g.generator.forward = record
            ref_pix.F = warp
            torch.manual_seed(seed)
            codes = g.generator.generate(cond, shape=[aud.shape[2], 2], batch_size=2 * P, aud_feat=aud, pre_latents=pre,
                                         pre_audio=aud_pre)
            ref_pix.F = TF
            g.generator.forward = fwd
            mp, mm = warp.margins()
            if min(mp, mm) >= MIN_MARGIN:
                break
            print("guided", case, "seed", seed, "margins %.3g %.3g: next seed" % (mp, mm), flush=True)
            seed += 100
        for layer, emb in zip(g.generator.layers, embs):
            layer.class_cond_embedding = emb
        for p in GREEDY:
            assert all(warp.unique_max[p]), "pair %d: a draw has tied maximum guided logits: choose another seed" % p
        assert torch.equal(codes[0::2], codes[1::2])
        T = codes.shape[1]
        kept = np.array(warp.kept, dtype=np.int32).reshape(P, T, 2)
        assert (kept >= 1).all()
        min_p, min_m = min(min_p, mp), min(min_m, mm)
        out["seed_%s" % case] = np.int64(seed)
        out["codes_%s" % case] = codes[0::2].numpy()
        out["kept_%s" % case] = np.ascontiguousarray(kept)
        print("guided", case, "seed", seed, codes[0::2, 0, 0].tolist(), "kept", kept.min(axis=(1, 2)).tolist(),
              "margins %.3g %.3g" % (mp, mm), flush=True)
    out["min_margin_top_p"] = np.float64(min_p)
    out["min_margin_min_p"] = np.float64(min_m)
    assert min(min_p, min_m) >= MIN_MARGIN
    np.savez_compressed(os.path.join(HERE, "guided.npz"), **out)


if __name__ == "__main__":
    main()
