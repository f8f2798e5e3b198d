"""s2g_body_vq — host mirror of nets/smplx_body_vq.py (inference): VQ-VAE encode -> quantise ->
decode round trip of ground-truth poses (BASELINE config 2)."""
from __future__ import annotations

import numpy as np
import torch

from ..data_utils.lower_body import c_index_3d, c_index_6d
from .base import resolve_device, shared_engine, strip_module


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
