"""Generate tests/golden/sampling.npz: codes and poses of the UNMODIFIED reference's s2g_body_pixel.infer_on_audio
(nets/smplx_body_pixel.py:232-289) under sampling controls.  Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_sampling.py

The reference has no sampling controls: GatedPixelCNN.generate draws ``F.softmax(logits).multinomial(1)``
(gated_pixelcnn_v2.py:173-176).  The module's ``F`` is swapped for a proxy whose ``softmax`` applies the warp of
ts_pixelcnn_sample (include/talkshow_b200.h) to the raw logits:
  - top_k: logits below the k-th largest (TopKLogitsWarper: ``l < topk(l, k).values[-1]``) -> -inf;
  - temperature t > 0: softmax(l / t) over the kept codes;
  - temperature 0 (greedy): the one-hot of the first-index argmax.
Everything else (the loop, the multinomial draw under the seed, the VQ decoders) is the reference's own code.  The codes
are captured from the generator's ``generate`` call inside infer_on_audio.  Running the script again reproduces the file
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

from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

SEED = 3100
POSE_STRIDE = 5   # poses are kept for every 5th frame (the codes, which determine them, are kept whole)
# (temperature, top_k); top_k is unused for greedy decoding
SETTINGS = [(0.7, 0), (1.3, 0), (1.0, 5), (0.8, 64), (0.0, 0)]
CASES = {   # geometry: (B, feature frames M -> T = M // 4 latent rows, speaker id, mfcc seed)
    "3d": (3, 300, 2, 3201),
    "6d": (2, 40, 1, 3202),
}


class WarpF:
    """torch.nn.functional with ``softmax`` replaced by the controlled warp (see the module docstring)."""

    def __init__(self, temperature, top_k):
        self.t, self.k = float(temperature), int(top_k)

    def __getattr__(self, name):
        return getattr(TF, name)

    def softmax(self, logits, dim=-1):
        if self.t == 0:
            return TF.one_hot(torch.argmax(logits, dim), logits.shape[dim]).to(logits.dtype)
        s = logits / self.t
        if 0 < self.k < logits.shape[dim]:
            kth = torch.topk(logits, self.k, dim).values[..., -1:]
            s = s.masked_fill(logits < kth, float("-inf"))
        return TF.softmax(s, dim)


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
        for i, (t, k) in enumerate(SETTINGS):
            ref_pix.F = WarpF(t, k)
            captured.clear()
            torch.manual_seed(SEED + i)
            pred = g.infer_on_audio("synthetic.wav", id=torch.tensor([spk]), fps=30, B=B)    # (B, 4T, C)
            ref_pix.F = TF
            out["codes_%s_%d" % (key, i)] = captured[0].numpy()
            out["poses_%s_%d" % (key, i)] = np.ascontiguousarray(np.asarray(pred, dtype=np.float32)[:, ::POSE_STRIDE])
            print("sampling", key, (t, k), captured[0][0, :4].tolist(), np.asarray(pred).shape, flush=True)
    np.savez_compressed(os.path.join(HERE, "sampling.npz"), **out)


if __name__ == "__main__":
    main()
