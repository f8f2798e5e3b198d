"""Generate tests/golden/style.npz: codes and per-draw log p of the UNMODIFIED reference's GatedPixelCNN.generate
(nets/spg/gated_pixelcnn_v2.py:152-177) conditioned on convex mixtures of the speaker embeddings (styled sampling,
ts_pixelcnn_sample_styled in include/talkshow_b200.h).  Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_style.py

Each layer's ``class_cond_embedding`` instance is swapped for ``BlendEmbedding``, which holds the same table and maps a
per-clip weight tensor w [B, ncls], passed to ``generate`` as the label, to the blend of the rule, in its fp32 order:
acc = w0 E[0], then acc = acc + w_s E[s] for s = 1 .. ncls-1 (separate elementwise products and sums, no contraction).
The rest of the network is the reference's.  The multinomial draw runs under a torch seed, as make_golden.py does for
pixel_b3_t75.npz, so the noise is ``draw_noise(2T, B)`` after ``torch.manual_seed(seed)``.  The module's ``F`` is
swapped for a proxy that records the reference's ``log_softmax`` of every call's logits; the log p of each draw is read
at the code the loop kept.

Every one-hot schedule is checked here against a plain labelled run of the reference (same seed): the codes and the
recorded log-softmax must agree exactly.

Only per-clip mixtures go through the unmodified forward: its ``h[:, :, None, None]`` broadcasts one class term over every
position, so a schedule that changes from row to row cannot be expressed through it.  Per-row schedules are pinned by the
oracle (tests/oracle_style.py) and by exact properties of the engine instead: one-hot rows equal the labelled call, the
rows before a switch equal the constant schedule, and the sampler's log p equals the styled teacher-forced scorer's.

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

from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

SEED = 6100
NCLS = 4
CASES = {   # geometry: (B, feature frames M -> T = M // 4 latent rows, mfcc seed)
    "3d": (3, 120, 6201),
    "6d": (2, 40, 6202),
}


def mixtures(B):
    """name -> per-clip weights [B, 4] float32"""
    out = {}
    for s in range(NCLS):
        w = np.zeros((B, NCLS), np.float32)
        w[:, s] = 1
        out["onehot%d" % s] = w
    rows = {"half02": [0.5, 0, 0.5, 0], "three1_13": [0, 0.75, 0, 0.25], "uniform": [0.25] * 4, "nine1_20": [0.1, 0, 0.9, 0]}
    for name, r in rows.items():
        out[name] = np.tile(np.array(r, np.float32), (B, 1))
    out["mixed"] = np.array([rows["half02"], rows["three1_13"], rows["uniform"]][:B], np.float32)
    return out


class BlendEmbedding(torch.nn.Module):
    """class_cond_embedding of a styled call: per-clip weights [B, ncls] -> [B, 2 dim] in the rule's fp32 order."""

    def __init__(self, emb):
        super().__init__()
        self.weight = emb.weight

    def forward(self, w):
        acc = w[:, 0:1] * self.weight[0]
        for s in range(1, self.weight.shape[0]):
            acc = acc + w[:, s:s + 1] * self.weight[s]
        return acc


class LogSoftmaxF:
    """torch.nn.functional that records log_softmax of every softmax call's logits."""

    def __init__(self):
        self.logsm = []

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        self.logsm.append(TF.log_softmax(logits, dim).numpy())
        return TF.softmax(logits, dim)


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
    for key, (B, M, mseed) in CASES.items():
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
        g.generator.eval()
        g.audioencoder.eval()
        mfcc = synth.synth_mfcc(B, M, seed=mseed)
        audio = g.audioencoder(mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)          # [B,256,T,2]
        plain = [layer.class_cond_embedding for layer in g.generator.layers]
        blend = [BlendEmbedding(e) for e in plain]

        def run(label, seed, styled):
            for layer, e in zip(g.generator.layers, blend if styled else plain):
                layer.class_cond_embedding = e
            proxy = LogSoftmaxF()
            ref_pix.F = proxy
            torch.manual_seed(seed)
            codes = g.generator.generate(label, shape=[T, 2], batch_size=B, aud_feat=audio).numpy()
            ref_pix.F = TF
            for layer, e in zip(g.generator.layers, plain):
                layer.class_cond_embedding = e
            logsm = np.stack(proxy.logsm, 0).reshape(T, 2, B, -1)                # one call per (row, column)
            logp = np.take_along_axis(logsm, codes.transpose(1, 2, 0)[..., None], -1)[..., 0].transpose(2, 0, 1)
            return codes, np.ascontiguousarray(logp, dtype=np.float32), logsm

        names, weights, seeds, codes_all, logp_all = [], [], [], [], []
        for ci, (name, w) in enumerate(mixtures(B).items()):
            seed = SEED + ci
            codes, logp, logsm = run(torch.from_numpy(w), seed, True)
            if name.startswith("onehot"):
                c_ref, _, l_ref = run(torch.full((B,), int(name[-1]), dtype=torch.int64), seed, False)
                assert (codes == c_ref).all() and np.array_equal(logsm, l_ref), "one-hot %s differs from its label" % name
            names.append(name)
            weights.append(w)
            seeds.append(seed)
            codes_all.append(codes)
            logp_all.append(logp)
            print("style", key, name, "seed", seed, codes[0, :3].tolist(), flush=True)
        out[key + "_mfcc"] = mfcc.numpy()
        out[key + "_audio"] = np.ascontiguousarray(audio[..., 0].numpy())
        out[key + "_cases"] = np.array(names)
        out[key + "_weights"] = np.stack(weights)
        out[key + "_seed"] = np.array(seeds, dtype=np.int64)
        out[key + "_codes"] = np.stack(codes_all)
        out[key + "_logp"] = np.stack(logp_all)
        out[key + "_fp"] = np.array(list(synth.fingerprint(bp).values()))
    np.savez_compressed(os.path.join(HERE, "style.npz"), **out)


if __name__ == "__main__":
    main()
