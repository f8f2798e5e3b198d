"""Generate tests/golden/eval_losses.npz: the held-out losses of a face / VQ / prior trio as the UNMODIFIED reference's own
modules and get_loss compute them, in eval mode, for a 3-D and a convert_to_6d ("6-D") trio of the seeded synthetic
checkpoints of talkshow_b200/synth.py.  Run on a host with a reference checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_eval.py

Per trio (key '3d' / '6d'), from one batch bat_3d() / bat_6d() (the inputs are regenerated from their seeds; their
fingerprints are stored as in_fp_<key>):
  face   s2g_face (:95-167): the generator in eval mode with time_steps = F passed explicitly (the reference sets it only in
         training mode), then the wrapper's get_loss -> 'MSELoss', 'exp_loss';
  vq     s2g_body_vq.vq_train (:155-206) restated for eval mode, where VQVAE.forward returns (e, recon) untransposed and
         get_loss would fail: encoder -> vq_layer (argmin + codebook rows) -> decoder, then the wrapper's get_loss with
         e_q_loss = commitment_cost * mse(z, e) -> 'brec_loss', 'bvelocity_loss', 'hrec_loss', 'hvelocity_loss';
  prior  s2g_body_pixel.__call__ with its modules in eval mode (make_golden_prior_ce.run_case) -> 'ce_loss'.
Also stored: the codes, the per-clip sums (fp64 over the reference's fp32 outputs) and strided slices of recon / pred.
Only eval_losses.npz is written.
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

LOSS_NAMES = ["MSELoss", "exp_loss", "brec_loss", "bvelocity_loss", "hrec_loss", "hvelocity_loss", "ce_loss"]
STRIDE = 8      # frames kept of recon / pred


def synth_expression(B, F, seed):
    """Expression coefficients [B,100,F]: uniform in [-0.5, 0.5), float64 math rounded once (host independent)."""
    gen = torch.Generator().manual_seed(seed + 13)
    return (torch.rand((B, 100, F), generator=gen, dtype=torch.float64) - 0.5).float()


def _bat(B, F, poses, seed, speakers):
    n = -(-F * 16000 // 30)                                  # samples of F frames at 30 fps
    return {"wave": synth.synth_wave(B, n, seed=seed), "aud_feat": synth.synth_mfcc(B, F, seed=seed + 1), "poses": poses,
            "expression": synth_expression(B, F, seed + 2), "speaker": torch.tensor(speakers)}


def bat_3d():
    """B = 2 clips of 120 frames (4 s, 30 latent rows), speakers 20 and 22."""
    return _bat(2, 120, synth.synth_poses(2, 120, seed=931), 932, [20, 22])


def bat_6d():
    """B = 2 clips of 88 frames in the 6-D pose layout [B,330,F] (two axis-angle-scale blocks stacked)."""
    poses = torch.cat([synth.synth_poses(2, 88, seed=941), synth.synth_poses(2, 88, seed=942)], 1)
    return _bat(2, 88, poses, 943, [23, 21])


def input_fingerprint(bat):
    return np.array([float(bat[k].double().sum()) for k in ("wave", "aud_feat", "poses", "expression")])


def main():
    import_reference()
    import nets.smplx_body_pixel as ref_bp
    import nets.smplx_body_vq as ref_vq
    import nets.smplx_face as ref_face
    import torch.nn.functional as F
    from trainer.config import load_JsonConfig

    from make_golden_prior_ce import run_case

    tmp = tempfile.mkdtemp()
    out = {"loss_names": np.array(LOSS_NAMES), "stride": STRIDE}
    for key, six, bat, face, vq, bp in (
            ("3d", False, bat_3d(), synth.face_checkpoint(0), synth.body_vq_checkpoint(0), synth.body_pixel_checkpoint(0)),
            ("6d", True, bat_6d(), synth.face_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0),
             synth.body_pixel_checkpoint_6d(0))):
        vq_path = os.path.join(tmp, "vq_%s.pth" % key)
        torch.save({"generator": vq}, vq_path)
        cfg = load_JsonConfig("config/body_pixel.json")
        cfg.Data.pose.convert_to_6d = six
        cfg.Model.vq_path = vq_path
        a = types.SimpleNamespace(gpu="cpu", infer=True)
        losses = {}
        B, nf = bat["poses"].shape[0], bat["poses"].shape[2]

        # ---- face ------------------------------------------------------------------------------------------------
        with torch.no_grad():
            gf = ref_face.TrainWrapper(a, cfg)
            gf.generator.load_state_dict(face["generator"], strict=True)
            gf.generator.eval()
            aud = bat["wave"][:, None, :].permute(0, 2, 1)                                 # bat['aud_feat'] of the face, :106
            gt = torch.cat([bat["poses"].permute(0, 2, 1), bat["expression"].permute(0, 2, 1)], 2)
            pred, _ = gf.generator(aud, gt, F.one_hot(bat["speaker"] - 20, 4), time_steps=nf)
            _, ld = gf.get_loss(pred_poses=pred, gt_poses=gt, pre_poses=None, aud=aud)
        losses.update({k: float(v) for k, v in ld.items()})
        out["clip_face_%s" % key] = np.stack([(pred[..., :6] - gt[..., :6]).abs().double().sum((1, 2)).numpy(),
                                              ((pred[..., -100:] - gt[..., -100:]) ** 2).double().sum((1, 2)).numpy()], 1)
        out["pred_%s" % key] = pred[:, ::STRIDE].numpy()

        # ---- VQ pair -----------------------------------------------------------------------------------------------
        gv = ref_vq.TrainWrapper(a, cfg)
        gv.load_state_dict(vq)
        gtp = bat["poses"][:, gv.c_index, :].permute(0, 2, 1)
        nb = gv.each_dim[1]
        with torch.no_grad():
            for name, model, part in (("b", gv.g_body, gtp[..., :nb]), ("h", gv.g_hand, gtp[..., nb:])):
                model.eval()
                z = model.encoder(part.transpose(1, 2))
                e, idx = model.vq_layer(z)
                recon = model.decoder(e)[0].transpose(1, 2)
                e_q = model.vq_layer.commitment_cost * F.mse_loss(z, e)
                _, ld = gv.get_loss(pred_poses=recon, gt_poses=part, e_q_loss=e_q)
                losses.update({name + k: float(v) for k, v in ld.items()})
                vr, vg = recon[:, 1:] - recon[:, :-1], part[:, 1:] - part[:, :-1]
                out["clip_%s_%s" % (name, key)] = np.stack([(recon - part).abs().double().sum((1, 2)).numpy(),
                                                            (vr - vg).abs().double().sum((1, 2)).numpy(),
                                                            ((z - e) ** 2).double().sum((1, 2)).numpy()], 1)
                out["e_q_%s_%s" % (name, key)] = np.float64(e_q)
                out["codes_%s_%s" % (name, key)] = idx.numpy()
                out["recon_%s_%s" % (name, key)] = recon[:, ::STRIDE].numpy()

        # ---- prior -------------------------------------------------------------------------------------------------
        ce, lat, _ = run_case(ref_bp, cfg, bp, bat)
        assert torch.equal(lat[..., 0], torch.from_numpy(out["codes_b_%s" % key]))
        losses["ce_loss"] = float(ce)

        out["losses_%s" % key] = np.array([losses[k] for k in LOSS_NAMES])
        out["in_fp_%s" % key] = input_fingerprint(bat)
        out["fp_%s" % key] = np.array([list(synth.fingerprint(c).values()) for c in (face, vq, bp)])
        print("eval", key, {k: round(v, 6) for k, v in losses.items()})
    np.savez_compressed(os.path.join(HERE, "eval_losses.npz"), **out)


if __name__ == "__main__":
    main()
