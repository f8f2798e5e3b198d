"""Generate tests/golden/prior_ce.npz: the body prior's cross-entropy ``ce_loss`` as the UNMODIFIED reference's
s2g_body_pixel.__call__(bat) computes it (nets/smplx_body_pixel.py:176-216), in validation mode.  Run on a host with a
reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_prior_ce.py

__call__ never puts its modules in eval mode, so the AudioEncoder's BatchNorm would use batch statistics and the
Dropout(0.1) of GatedPixelCNN.forward (gated_pixelcnn_v2.py:139-141) would be active; the generator and the audio
encoder are switched to eval() first, which is what s2g_body_pixel.evaluate restates.  __call__ steps the optimizers
after the loss, so every case uses a fresh wrapper.  Only prior_ce.npz is written; the other fixtures stay as
tests/golden/make_golden.py wrote them.
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

from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

LOGIT_ROWS = [0, 5, 21]


def bat_3d():
    """B = 3 clips of 88 frames (22 latent rows), speakers 20, 21, 23 (ids 0, 1, 3)."""
    return {"aud_feat": synth.synth_mfcc(3, 88, seed=901), "poses": synth.synth_poses(3, 88, seed=902),
            "speaker": torch.tensor([20, 21, 23])}


def bat_6d():
    """B = 2 clips of 88 frames in the 6-D pose layout (330 channels, indexed by c_index_6d)."""
    poses = torch.cat([synth.synth_poses(2, 88, seed=911), synth.synth_poses(2, 88, seed=912)], 1)
    return {"aud_feat": synth.synth_mfcc(2, 88, seed=913), "poses": poses, "speaker": torch.tensor([22, 20])}


def run_case(ref_bp, cfg, ckpt, bat):
    a = types.SimpleNamespace(gpu="cpu", infer=False)
    g = ref_bp.TrainWrapper(a, cfg)
    g.load_state_dict(ckpt)
    g.generator.eval()
    g.audioencoder.eval()
    g.g_body.eval()                             # as __call__ does (:192-194): a VQ layer in training mode updates its EMA
    g.g_hand.eval()
    # the codes and the teacher-forced logits the loss is taken over, recomputed through the same modules (:187-208)
    with torch.no_grad():
        gt = bat["poses"][:, g.c_index, :].permute(0, 2, 1)
        _, body = g.g_body.encode(gt_poses=gt[..., :g.each_dim[1]])
        _, hand = g.g_hand.encode(gt_poses=gt[..., g.each_dim[1]:])
        lat = torch.cat([body.unsqueeze(-1), hand.unsqueeze(-1)], -1)
        audio = g.audioencoder(bat["aud_feat"], frame_num=lat.shape[1] * 4).unsqueeze(-1).repeat(1, 1, 1, 2)
        logits = g.generator(lat, bat["speaker"] - 20, audio)
    _, loss_dict = g(bat)                       # ce_loss is taken before the optimizer step
    return loss_dict["ce_loss"], lat, logits


def main():
    import_reference()
    import nets.smplx_body_pixel as ref_bp
    from trainer.config import load_JsonConfig

    tmp = tempfile.mkdtemp()
    out = {}
    for key, ck, vq, six, bat in (("3d", synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), False, bat_3d()),
                                  ("6d", synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0), True, bat_6d())):
        vq_path = os.path.join(tmp, "vq_%s.pth" % key)
        torch.save({"generator": vq}, vq_path)
        cfg = load_JsonConfig("config/body_pixel.json")
        cfg.Data.pose.convert_to_6d = six
        cfg.Model.vq_path = vq_path
        ce, lat, logits = run_case(ref_bp, cfg, ck, bat)
        out["ce_%s" % key] = np.float64(ce)
        out["codes_%s" % key] = lat.numpy()
        out["logits_%s" % key] = logits[:, :, LOGIT_ROWS, :].numpy()
        out["in_fp_%s" % key] = np.array([float(bat["aud_feat"].double().sum()), float(bat["poses"].double().sum())])
        out["fp_%s" % key] = np.array(list(synth.fingerprint(ck).values()))
        print("prior_ce", key, ce, lat[0, :4].tolist())
    np.savez_compressed(os.path.join(HERE, "prior_ce.npz"), logit_rows=np.array(LOGIT_ROWS), **out)


if __name__ == "__main__":
    main()
