"""TEST INFRASTRUCTURE: held-out scoring on the CPU oracle, built on oracle/talkshow_oracle.py and tests/oracle_6d.py.

  vq_eval / face_eval   the forward half of s2g_body_vq.vq_train (nets/smplx_body_vq.py:155-206) and s2g_face.__call__
                        (nets/smplx_face.py:95-167) in eval mode, with the per-clip sums the engine returns (fp64 over the
                        fp32 outputs);
  vq_get_loss / face_get_loss
                        the reference's get_loss reductions (torch.mean over fp32, as the reference takes them);
  EvalOracleEngine      OracleEngine plus Engine.vq_score / face_score / pixelcnn_score / face_dim answered by the above,
                        so the wrappers' evaluate() and WholeBody.evaluate run on a machine without a GPU.
Never imported by the package."""
import torch
import torch.nn.functional as F

import oracle_6d as O6
import talkshow_oracle as O
from oracle_engine import OracleEngine

COMMITMENT_COST = 0.25


def vq_eval(sd, gt):
    """gt [B,F,C] -> (idx [B,T], recon [B,F,C], clip [B,3] float64, e_q_loss): encoder -> argmin -> decoder on the
    codebook rows; clip = per-clip sums of |recon - gt|, |d recon - d gt| and ||z - e||^2."""
    z = O.encoder_trunk(sd, "encoder.", gt.transpose(1, 2))
    z = F.conv1d(z, sd["encoder.pre_vq_conv.weight"], sd["encoder.pre_vq_conv.bias"])
    x = z.permute(0, 2, 1).contiguous()
    idx = O.vq_code_indices(sd, x.reshape(-1, x.shape[-1])).view(x.shape[0], x.shape[1])
    e = F.embedding(idx, sd["vq_layer.embeddings"]).permute(0, 2, 1).contiguous()
    recon = O.vq_decoder(sd, e).transpose(1, 2)
    vr, vg = recon[:, 1:] - recon[:, :-1], gt[:, 1:] - gt[:, :-1]
    clip = torch.stack([(recon - gt).abs().double().sum((1, 2)), (vr - vg).abs().double().sum((1, 2)),
                        ((z - e) ** 2).double().sum((1, 2))], 1)
    return idx, recon, clip, float(COMMITMENT_COST * F.mse_loss(z, e))


def vq_get_loss(recon, gt):
    """nets/smplx_body_vq.py:186-189 -> (rec_loss, velocity_loss)."""
    v_pr, v_gt = recon[:, 1:] - recon[:, :-1], gt[:, 1:] - gt[:, :-1]
    return float(torch.mean(torch.abs(recon - gt))), float(torch.mean(torch.abs(v_pr - v_gt)))


def face_eval(sd, wave, id_onehot, gt):
    """wave [B,N], gt [B,F,C] -> (pred [B,F,jaw+100] at frame = F, clip [B,2] float64: per-clip sums of
    |pred[..,:6] - gt[..,:6]| and (pred[..,-100:] - gt[..,-100:])^2)."""
    pred = O6.face_forward(sd, wave, id_onehot, gt.shape[1])
    clip = torch.stack([(pred[..., :6] - gt[..., :6]).abs().double().sum((1, 2)),
                        ((pred[..., -100:] - gt[..., -100:]) ** 2).double().sum((1, 2))], 1)
    return pred, clip


def face_get_loss(pred, gt):
    """nets/smplx_face.py:155-157 -> (MSELoss, exp_loss)."""
    return (float(torch.mean(torch.abs(pred[:, :, :6] - gt[:, :, :6]))),
            float(torch.mean((pred[:, :, -100:] - gt[:, :, -100:]) ** 2)))


class EvalOracleEngine(OracleEngine):
    @property
    def face_dim(self):
        sd = self.sd.get("face")
        return 0 if sd is None else int(sd["final_out.0.weight"].shape[0] + sd["final_out.1.weight"].shape[0])

    def face_forward(self, wave, id_onehot, frame):
        wave = wave.float().reshape(wave.shape[0], -1)
        return O6.face_forward(self.sd["face"], wave, id_onehot.float().expand(wave.shape[0], -1), frame)

    def vq_score(self, which, poses, want_recon=False):
        if poses.dim() != 3 or poses.shape[2] != self.vq_dim(which) or poses.shape[1] < 4 or poses.shape[1] % 4:
            raise ValueError("vq_score: poses %s" % (tuple(poses.shape),))
        idx, recon, clip, _ = vq_eval(self.sd["vq%d" % which], poses.float())
        return idx, clip, (recon if want_recon else None)

    def face_score(self, wave, id_onehot, gt, want_pred=False):
        if gt.dim() != 3 or gt.shape[2] < 100 or gt.shape[0] != wave.shape[0]:
            raise ValueError("face_score: wave %s, gt %s" % (tuple(wave.shape), tuple(gt.shape)))
        wave = wave.float().reshape(wave.shape[0], -1)
        pred, clip = face_eval(self.sd["face"], wave, id_onehot.float().expand(wave.shape[0], -1), gt.float())
        return clip, (pred if want_pred else None)

    def pixelcnn_score(self, aud, label, codes, want_logits=False):
        label = label.reshape(-1).to(torch.int64).expand(aud.shape[0])
        logits = O.pixelcnn_forward(self.sd["pixelcnn"], codes, label, aud.float().unsqueeze(-1).repeat(1, 1, 1, 2))
        nll = F.cross_entropy(logits, codes, reduction="none")
        return (nll, logits) if want_logits else nll
