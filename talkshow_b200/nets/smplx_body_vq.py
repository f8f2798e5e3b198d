"""s2g_body_vq — host mirror of nets/smplx_body_vq.py (inference): VQ-VAE encode -> quantise ->
decode round trip of ground-truth poses (BASELINE config 2)."""
from __future__ import annotations

import numpy as np
import torch

from ..data_utils.lower_body import c_index_3d, c_index_6d
from .base import resolve_device, shared_engine, strip_module


COMMITMENT_COST = 0.25   # VQVAE(..., commitment_cost=0.25), nets/spg/vqvae_1d.py:171-181


def score_vq_pair(engine, gt, n_body):
    """vq_train + get_loss of the body and the hand VQ-VAE (nets/smplx_body_vq.py:145-148,155-206) in eval mode.
    gt [B,F,C] (c_index applied; body columns first, n_body of them) ->
    (codes [B,T,2], {'brec_loss', 'bvelocity_loss', 'hrec_loss', 'hvelocity_loss'} as floats, per-clip float64 values of
    those four and of 'be_q_loss' / 'he_q_loss' = commitment_cost * mean ||z - e||^2, the term the reference leaves out
    of its dict)."""
    B, F = gt.shape[:2]
    losses, per_clip, codes = {}, {}, []
    for name, which, part in (("b", 0, gt[..., :n_body]), ("h", 1, gt[..., n_body:])):
        idx, clip, _ = engine.vq_score(which, part.contiguous())
        clip = clip.cpu()
        C, T = part.shape[2], idx.shape[1]
        per_clip[name + "rec_loss"] = clip[:, 0] / (F * C)
        per_clip[name + "velocity_loss"] = clip[:, 1] / ((F - 1) * C)
        per_clip[name + "e_q_loss"] = COMMITMENT_COST * clip[:, 2] / (T * 64)
        losses[name + "rec_loss"] = float(clip[:, 0].sum() / (B * F * C))
        losses[name + "velocity_loss"] = float(clip[:, 1].sum() / (B * (F - 1) * C))
        codes.append(idx)
    return torch.stack(codes, -1), losses, per_clip


def check_pose_block(poses, convert_to_6d, who):
    """[B,165,F] (axis-angle) or [B,330,F] (convert_to_6d) with F a positive multiple of 4, else ValueError."""
    rows = 330 if convert_to_6d else 165
    if poses.dim() != 3 or poses.shape[1] != rows:
        raise ValueError("%s: poses %s, expected [B,%d,F] (convert_to_6d=%s)" % (who, tuple(poses.shape), rows, convert_to_6d))
    if poses.shape[2] < 4 or poses.shape[2] % 4:
        # the decoder returns 4 * (latent rows) frames: the reference fails on the recon / gt shape mismatch
        raise ValueError("%s: %d pose frames, the VQ-VAE scores multiples of 4" % (who, poses.shape[2]))


class TrainWrapper:
    def __init__(self, args, config, engine=None):
        self.args = args
        self.config = config
        self.device = resolve_device(self.args.gpu)
        self.convert_to_6d = self.config.Data.pose.convert_to_6d
        self.expression = self.config.Data.pose.expression
        self.num_classes = 4
        self.composition = self.config.Model.composition
        if not self.composition:
            raise NotImplementedError("talkshow_b200 builds the composition=true VQ-VAE pair (config/body_vq.json)")
        scale = 2 if self.convert_to_6d else 1                                   # nets/smplx_body_vq.py:96-126
        self.each_dim = [0, 39 * scale, 90 * scale, 100 if self.expression else 0]
        self.c_index = c_index_6d if self.convert_to_6d else c_index_3d
        self.engine = engine or shared_engine(self.device)

    def load_state_dict(self, state_dict):
        """{'g_body': sd, 'g_hand': sd} (nets/smplx_body_vq.py:297-302).  Like the reference's strict load, VQ-VAEs whose
        pose channels are not the config's (39 / 90, or 78 / 180 with convert_to_6d) raise RuntimeError."""
        self._loaded = {"g_body": strip_module(state_dict["g_body"]), "g_hand": strip_module(state_dict["g_hand"])}
        self.engine.load_vq(0, self._loaded["g_body"])
        self.engine.load_vq(1, self._loaded["g_hand"])
        got = [self.engine.vq_dim(0), self.engine.vq_dim(1)]
        if got != self.each_dim[1:3]:
            raise RuntimeError("s2g_body_vq: the checkpoint's VQ-VAEs have %s pose channels, the config (convert_to_6d=%s) "
                               "builds %s" % (got, self.convert_to_6d, self.each_dim[1:3]))

    def state_dict(self):
        """nets/smplx_body_vq.py:77-94 (composition): the loaded weights in the layout the reference saves; optimizer and
        discriminator slots empty."""
        loaded = getattr(self, "_loaded", {"g_body": None, "g_hand": None})
        return {"g_body": loaded["g_body"], "g_body_optim": None, "g_hand": loaded["g_hand"], "g_hand_optim": None,
                "discriminator": None, "discriminator_optim": None}

    def evaluate(self, bat):
        """The forward half of the reference's training step __call__(bat) (:128-206) in eval mode, which the reference
        itself cannot run (in eval VQVAE.forward returns (e, recon) untransposed and get_loss fails): encoder -> argmin
        quantisation -> decoder on the codebook rows (no straight-through add) -> get_loss.  bat: 'poses' [B,165,F], or
        [B,330,F] with convert_to_6d; F a multiple of 4.  Returns (None, {'brec_loss', 'bvelocity_loss', 'hrec_loss',
        'hvelocity_loss'}); per-clip values, the commitment terms included, are kept as self.last_losses and the codes
        [B,T,2] as self.last_codes."""
        poses = torch.as_tensor(bat["poses"]).to(torch.float32)
        check_pose_block(poses, self.convert_to_6d, "s2g_body_vq.evaluate")
        gt = poses[:, self.c_index, :].permute(0, 2, 1)
        self.last_codes, losses, self.last_losses = score_vq_pair(self.engine, gt, self.each_dim[1])
        return None, losses

    def encode(self, initial_pose):
        """initial_pose (B,165,F), (B,330,F) with convert_to_6d -> (idx_body [B,T], idx_hand [B,T]) int64 on the device."""
        gt = initial_pose.to(torch.float32)[:, self.c_index].permute(0, 2, 1).contiguous()
        nb = self.each_dim[1]
        ib = self.engine.vq_encode(0, gt[..., :nb].contiguous())
        ih = self.engine.vq_encode(1, gt[..., nb:].contiguous())
        return ib, ih

    def infer_on_audio(self, aud_fn, initial_pose=None, norm_stats=None, exp=None, var=None, w_pre=False,
                       continuity=False, id=None, fps=15, sr=22000, smooth=False, **kwargs):
        """initial_pose (B,165,F) -> numpy (F, B*129); (B,330,F) -> (F, B*258) with convert_to_6d
        (nets/smplx_body_vq.py:208-295; the audio
        argument is unused by the reference's VQ path too)."""
        assert self.args.infer, "train mode"
        if self.config.Data.pose.normalization:
            raise NotImplementedError("normalised VQ outputs are outside the built path (config/body_vq.json: false)")
        if continuity:
            # :256-271: five 60-frame chunks, each encoded/quantised/decoded on its own (pre_state is ignored by
            # Decoder.forward, vqvae_1d.py:139-149) and concatenated along time
            bs, hs = [], []
            for i in range(5):
                ib, ih = self.encode(initial_pose[:, :, i * 60:(i + 1) * 60])
                bs.append(self.engine.vq_decode(0, ib))
                hs.append(self.engine.vq_decode(1, ih))
            body, hand = torch.cat(bs, 2), torch.cat(hs, 2)
        else:
            ib, ih = self.encode(initial_pose)
            body = self.engine.vq_decode(0, ib)
            hand = self.engine.vq_decode(1, ih)
        output = torch.cat([body, hand], 1).transpose(1, 2).cpu().numpy()          # (B,F,129) / (B,F,258)
        if smooth:                                                                  # :283-291
            lamda, smooth_f, frame = 0.8, 10, 149
            for i in range(smooth_f):
                f = frame + i
                l = lamda * (i + 1) / smooth_f
                output[0, f] = (1 - l) * output[0, f - 1] + l * output[0, f]
        return np.concatenate(output, axis=1)
