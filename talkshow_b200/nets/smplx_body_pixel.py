"""s2g_body_pixel — host mirror of the reference wrapper nets/smplx_body_pixel.py (inference
methods).  Audio features -> AudioEncoder -> gated-PixelCNN sampler -> two VQ-VAE decoders, all
inside the CUDA engine (C ABI: ts_body_generate / ts_pixelcnn_generate / ts_vq_decode)."""
from __future__ import annotations

import os

import numpy as np
import torch

from ..data_utils.lower_body import c_index_3d, c_index_6d
from ..data_utils.utils import get_mfcc_sepa, get_mfcc_ta, load_wav
from ..engine import (check_clip_controls, guide_kwargs, check_sample_controls, check_style, per_clip, resolve_clip_seeds, sample_controls,
                      sampled, shaping_kwargs)
from .base import draw_sampler_noise, resolve_device, shared_engine, strip_module


class TrainWrapper:
    """Constructor/attribute surface of nets/smplx_body_pixel.py:30-75 (args.gpu, args.infer,
    config.Data.pose.*, config.Model.{composition,bh_model,code_num,vq_path})."""

    def __init__(self, args, config, engine=None):
        self.args = args
        self.config = config
        self.device = resolve_device(self.args.gpu)
        self.global_step = 0
        self.convert_to_6d = self.config.Data.pose.convert_to_6d
        self.expression = self.config.Data.pose.expression
        self.epoch = 0
        self.init_params()
        self.num_classes = 4
        self.audio = True
        self.composition = self.config.Model.composition
        self.bh_model = self.config.Model.bh_model
        if not self.bh_model or not self.composition:
            raise NotImplementedError("talkshow_b200 builds the bh_model=true, composition=true prior "
                                      "(config/body_pixel.json); convert_to_6d selects the dim 512 x 10-layer geometry")
        self.c_index = c_index_6d if self.convert_to_6d else c_index_3d      # :72-75
        self.engine = engine or shared_engine(self.device)
        self.noise_device = self.device      # 'cpu' reproduces the CPU reference's RNG stream
        self.noise_per_step = True
        self.device_mfcc = True              # MFCC features on the device (ts_mfcc); False = host torchaudio chain
        # the reference loads the VQ-VAE checkpoint at construction (:59-62); honour it when present
        vq_path = getattr(self.config.Model, "vq_path", None)
        if vq_path and os.path.exists(vq_path):
            ck = torch.load(vq_path, map_location="cpu")["generator"]
            self.load_vq_state_dict(ck)

    def init_params(self):
        """nets/smplx_body_pixel.py:144-174: body 39 + hands 90 axis-angle dims, doubled for the 6-D layout
        (convert_to_6d: the prior is pixelcnn(2048, 512, 10, ...) instead of (2048, 256, 15, ...), :49-52)."""
        scale = 2 if self.convert_to_6d else 1
        body, hand = 39 * scale, 90 * scale
        self.each_dim = [0, body, hand, 100 if self.expression else 0]
        self.dim_list = [0, 0, 0, body, body + hand]
        self.full_dim = body + hand
        self.pose = int(self.full_dim / round(3 * scale))

    # -- checkpoints -----------------------------------------------------------------------------
    def load_vq_state_dict(self, sd):
        """{'g_body': ..., 'g_hand': ...} as saved by s2g_body_vq.state_dict()."""
        self.engine.load_vq(0, strip_module(sd["g_body"]))
        self.engine.load_vq(1, strip_module(sd["g_hand"]))

    def load_state_dict(self, state_dict):
        """ckpt['generator'] of a body-pixel checkpoint (nets/smplx_body_pixel.py:115-142)."""
        sd = {k: (strip_module(v) if v is not None else None) for k, v in state_dict.items() if isinstance(v, dict) or v is None}
        gen = sd["generator"] if "generator" in sd else strip_module(state_dict)
        self.engine.load_pixelcnn(gen)
        self._loaded = {"generator": gen, "audioencoder": None}
        if sd.get("audioencoder") is not None:
            self.engine.load_audioenc(sd["audioencoder"])
            self._loaded["audioencoder"] = sd["audioencoder"]

    def state_dict(self):
        """The nested layout the reference saves (nets/smplx_body_pixel.py:104-113): the weights that were loaded (the engine
        keeps repacked copies only), optimizer / discriminator slots empty — this is an inference engine."""
        loaded = getattr(self, "_loaded", {"generator": None, "audioencoder": None})
        return {"generator": loaded["generator"], "generator_optim": None, "audioencoder": loaded["audioencoder"],
                "audioencoder_optim": None, "discriminator": None, "discriminator_optim": None}

    # -- evaluation ------------------------------------------------------------------------------
    def evaluate(self, bat):
        """The forward half of the reference's training step __call__(bat) (:183-216) in validation mode (BatchNorm
        running statistics, dropout off): ground-truth poses -> VQ codes, audio features -> AudioEncoder, one
        teacher-forced prior forward over all rows, cross-entropy against the codes.  bat: 'aud_feat' [B,64,M],
        'poses' [B,C,F] (165 axis-angle channels, or the 6-D layout), 'speaker' [B] (id = speaker - 20).
        Returns (None, {'ce_loss': float}); the per-position NLL [B,T,2] is kept as self.last_nll."""
        aud = bat["aud_feat"].to(torch.float32)
        poses = bat["poses"].to(torch.float32)
        label = (torch.as_tensor(bat["speaker"]) - 20).reshape(-1).to(torch.int64)
        gt = poses[:, self.c_index, :].permute(0, 2, 1)                       # [B,F,C]
        nb = self.each_dim[1]
        body = self.engine.vq_encode(0, gt[..., :nb].contiguous())
        hand = self.engine.vq_encode(1, gt[..., nb:].contiguous())
        latents = torch.stack([body, hand], -1)                               # [B,T,2]
        audio = self.engine.audio_encode(aud)                                 # [B,256,Ta]
        if audio.shape[2] != latents.shape[1]:
            # the reference fails in the prior's concatenation of code and audio rows (gated_pixelcnn_v2.py:143)
            raise ValueError("evaluate: %d audio rows (%d feature frames) vs %d code rows (%d pose frames)"
                             % (audio.shape[2], aud.shape[2], latents.shape[1], poses.shape[2]))
        nll = self.engine.pixelcnn_score(audio, label, latents)
        self.last_nll = nll
        return None, {"ce_loss": float(nll.double().mean())}

    # -- inference -------------------------------------------------------------------------------
    def _noise(self, T, B):
        return draw_sampler_noise(T, B, self.noise_device, per_step=self.noise_per_step)

    def infer_on_audio(self, aud_fn, initial_pose=None, norm_stats=None, exp=None, var=None, w_pre=False, rand=None,
                       continuity=False, id=None, fps=15, sr=22000, B=1, am=None, am_sr=None, frame=0, **kwargs):
        """(aud_fn) -> generated motion, numpy (B, F, 129).  Reference: :232-289.  Guidance as in ``generate``
        (``guidance``, ``guide_id``, ``guide_style``); ``guide_audio`` is "silence" or (M, 64) features like an array
        ``aud_fn``.  Not with ``continuity``."""
        assert self.args.infer, "train mode"
        ctl = {k: kwargs[k] for k in ("temperature", "top_k", "keep_logp", "top_p", "min_p", "clip_seeds", "repetition_penalty",
                                      "repetition_window", "code_bias") if k in kwargs}
        if kwargs.get("guidance") is not None:
            if continuity:
                raise ValueError("infer_on_audio: guidance is not supported with continuity=True (the clip is cut into "
                                 "two chunks); guide each chunk through infer()")
            ga = kwargs.get("guide_audio")
            if ga is not None and not isinstance(ga, str):
                ga = torch.from_numpy(np.ascontiguousarray(np.asarray(ga, dtype=np.float32).T))[None].repeat(B, 1, 1)
            ctl.update(guidance=kwargs["guidance"], guide_mfcc=ga, guide_id=kwargs.get("guide_id"),
                       guide_style=kwargs.get("guide_style"))
        if kwargs.get("noise_fn") is not None and kwargs.get("clip_seeds") is not None:
            raise ValueError("infer_on_audio: noise_fn and clip_seeds are two noise sources; give one")
        if kwargs.get("anchors") is not None:
            if continuity:
                raise ValueError("infer_on_audio: anchors are not supported with continuity=True (the clip is cut into "
                                 "two chunks); anchor each chunk through infer()")
            ctl["anchors"] = kwargs["anchors"]
        if kwargs.get("style") is not None:
            ctl["style"] = kwargs["style"]
        if continuity:
            return self._infer_continuity(aud_fn, id, fps, sr, B, **ctl)
        if torch.is_tensor(aud_fn) or isinstance(aud_fn, np.ndarray):
            aud_feat = np.asarray(aud_fn, dtype=np.float32)          # already (M, 64) features
            mfcc = torch.from_numpy(np.ascontiguousarray(aud_feat.T))[None].repeat(B, 1, 1)   # [B,64,M]
        elif fps == 30 and sr == 22000 and self.device_mfcc:
            audio, sr_0 = load_wav(aud_fn)                           # decode on the host, features on the device
            mfcc = self.engine.mfcc(audio.mean(0, keepdim=True), sr_0).repeat(B, 1, 1)
        else:
            aud_feat = get_mfcc_ta(aud_fn, sr=sr, fps=fps, smlpx=True, type="mfcc", am=am)
            mfcc = torch.from_numpy(np.ascontiguousarray(aud_feat.T))[None].repeat(B, 1, 1)
        label = torch.tensor([0]) if id is None else id.reshape(-1).repeat(B)[:B] if id.numel() == 1 else id
        return self.generate(mfcc, label, noise_fn=kwargs.get("noise_fn"), **ctl).cpu().numpy()

    def generate(self, aud, id, frame_num=0, noise_fn=None, temperature=1.0, top_k=0, keep_logp=False, top_p=1.0, min_p=0.0,
                 clip_seeds=None, anchors=None, style=None, repetition_penalty=1.0, repetition_window=8, code_bias=None,
                 guidance=None, guide_mfcc=None, guide_id=None, guide_style=None):
        """tensor API (:306-326): aud [B,64,M] features, id [B] -> torch (B, F, 129) on the device.
        (The reference's version passes decode()'s tuple to torch.cat and raises; this returns the
        tensor its infer_on_audio builds.)

        Sampling controls of the prior (Engine.pixelcnn_generate): ``temperature`` (0 = greedy decoding, which draws no
        noise), ``top_k`` (0 = off); ``keep_logp`` keeps each draw's log-likelihood under the untempered prior as
        self.last_logp [B,T,2].  ``top_p`` (1 = off) and ``min_p`` (0 = off) add nucleus and min-p truncation; with
        ``keep_logp`` the number of codes each such draw chose among is kept as self.last_kept [B,T,2] (None when both are
        off).  The defaults draw exactly like the reference.

        ``clip_seeds``: seeded sampling instead of torch-stream noise, so that a clip's motion depends only on its own seed
        (not on B or its place in the batch).  An integer s seeds clip b with s + b (``engine.clip_seeds``); a length-B
        sequence or int64 tensor gives each clip its seed.  Not combinable with ``noise_fn``.

        ``anchors`` [B,T,2] (T latent rows; int64 tensor or integer numpy array): a code in [0, 2048) pins that draw,
        -1 samples it (Engine.pixelcnn_generate).  The codes of the call, pinned and drawn, are kept as self.last_codes.
        To keep part of a known motion: ``torch.stack(vq.encode(poses), -1)`` of an s2g_body_vq, with -1 where new motion
        is wanted.  The prior is causal: a pinned code conditions the draws after it, not those before.

        ``style`` [B,T,4] per-row or [B,4] per-clip speaker weights (Engine.check_style: convex mixtures, float): the
        prior is conditioned on that mixture of its speaker embeddings instead of ``id``, which is then not read.  A
        one-hot row of speaker s is exactly ``id = s``; a fade between two one-hot rows changes style over those rows.

        Per-clip controls: ``temperature``, ``top_k``, ``top_p`` and ``min_p`` each take a scalar or one value per clip (a
        length-B sequence, 1-D array or tensor; Engine.pixelcnn_generate), so one batch serves clips with different
        settings; clip b draws what it draws alone under its own values.  Noise is drawn when any clip samples.

        Logit shaping (Engine.pixelcnn_generate): ``repetition_penalty`` (>= 1, 1 = off; scalar or per clip) penalises the
        codes the clip drew at the same column in its last ``repetition_window`` latent rows (8 rows, about 1 s), which
        breaks the loops greedy or cold sampling falls into; ``code_bias`` [2,2048] or [B,2,2048] is added to the logits
        (column 0 body codes, column 1 hand codes; -inf never draws the code).

        Guidance (Engine.body_generate): ``guidance`` w (scalar or per clip, in [0, 100]; 1 = none) pushes every draw
        away from a negative conditioning: ``guide_mfcc`` [B,64,M] or "silence" (audio guidance: gestures that follow the
        speech more closely), ``guide_id`` [B] (another speaker) and / or ``guide_style`` (e.g. a uniform blend).  Fields
        not given copy the clip's own.  The prior was trained without condition dropout, so this is contrastive guidance
        against the chosen conditioning.  With ``keep_logp`` the negative branches' log p is kept as
        self.last_guide_logp."""
        mfcc = aud.to(torch.float32)
        B, _, M = mfcc.shape
        T = self.engine.latent_rows(M)
        seeds = self._seeds(clip_seeds, B, noise_fn)
        shaping = shaping_kwargs(repetition_penalty, repetition_window, code_bias, B)
        guide = guide_kwargs(guidance, guide_mfcc, guide_id, guide_style, keep_logp, self.engine, B, M)
        noise = self._draw_noise(T, B, noise_fn, temperature, top_k, top_p, min_p, seeds)
        ctl = sample_controls(temperature, top_k, keep_logp, top_p, min_p)
        ctl.update(shaping)
        if noise is None and seeds is not None and sampled(temperature):
            ctl["seeds"] = seeds
        if anchors is not None:
            ctl["anchors"] = anchors
        if style is not None:
            ctl["style"] = style
        ctl.update(guide)
        out = self.engine.body_generate(mfcc, id.to(torch.int64), noise, **ctl)
        self.last_codes, poses = out[0], out[1]
        self.last_logp = out[2] if keep_logp else None
        self.last_kept = out[3] if ctl.get("want_kept") else None
        self.last_guide_logp = out[-1] if guide and keep_logp else None
        return poses

    def _draw_noise(self, T, B, noise_fn, temperature, top_k, top_p=1.0, min_p=0.0, seeds=None):
        """[2T,B,2048] Exp(1) draws (RNG contract), or None for greedy decoding (every clip greedy) and seeded sampling
        (controls validated first, per clip when given per clip)."""
        if per_clip(temperature, top_k, top_p, min_p):
            check_clip_controls(temperature, top_k, top_p, min_p, B)
        else:
            check_sample_controls(temperature, top_k, top_p, min_p)
        if not sampled(temperature) or seeds is not None:
            return None
        return self._noise(T, B) if noise_fn is None else noise_fn(T, B)

    @staticmethod
    def _seeds(clip_seeds, B, noise_fn):
        """``clip_seeds`` as int64 [B] (or None); ValueError with a noise_fn as well."""
        if clip_seeds is not None and noise_fn is not None:
            raise ValueError("noise_fn and clip_seeds are two noise sources; give one")
        return resolve_clip_seeds(clip_seeds, B)

    def infer(self, aud_feat, frame, id, B, pre_latents=None, pre_audio=None, pre_pose=None, noise_fn=None,
              temperature=1.0, top_k=0, keep_logp=False, top_p=1.0, min_p=0.0, clip_seeds=None, anchors=None, style=None,
              repetition_penalty=1.0, repetition_window=8, code_bias=None, guidance=None, guide_mfcc=None, guide_id=None,
              guide_style=None, guide_pre_audio=None):
        """The reference's inner call (:291-304): aud_feat [B,M,64] (time-major features of ONE chunk) ->
        (latents [B,T,2], audio [B,256,T,2], body [B,39,4T], hand [B,90,4T]).  ``pre_latents`` / ``pre_audio`` (the first
        two results of the previous chunk's call) condition the sampler on that chunk (GatedPixelCNN.generate :158-165);
        ``pre_pose`` is accepted and unused like in the reference, whose Decoder.forward ignores ``pre_state``
        (nets/spg/vqvae_1d.py:139-149) — each chunk is decoded on its own.  Sampling controls as in ``generate``; with
        ``keep_logp`` the chunk's logp [B,T,2] is kept as self.last_logp (and its keep-set sizes as self.last_kept).
        ``clip_seeds`` as in ``generate``; with ``pre_latents`` the chunk's draws are keyed by their absolute rows (after
        the T0 rows of the previous chunk), so a seeded clip's noise does not depend on where it is cut into chunks.
        ``anchors`` [B,T,2] cover this chunk's T rows (as in ``generate``); with ``pre_latents`` they pin rows after the
        prefix.  ``style`` [B,T0+T,4] (or [B,4]) as in ``generate``, its rows covering the prefix and the chunk.  Per-clip
        controls and logit shaping as in ``generate``; with ``pre_latents`` the repetition window reaches back into the
        prefix's codes.  Guidance as in ``generate``, with ``guide_mfcc`` [B,M,64] (time-major like ``aud_feat``) or
        "silence"; with ``pre_latents`` the negative branch's prefix audio is ``guide_pre_audio`` (default: the clip's
        ``pre_audio``), and both branches are fed the prefix codes."""
        a = self.engine.audio_encode(aud_feat.transpose(1, 2).contiguous())            # [B,256,T]
        T = a.shape[2]
        label = id.reshape(-1)
        seeds = self._seeds(clip_seeds, B, noise_fn)
        shaping = shaping_kwargs(repetition_penalty, repetition_window, code_bias, B)
        if isinstance(guide_mfcc, str):   # "silence" (guide_kwargs refuses any other name): [B,64,M] from the front end
            gmc = guide_mfcc if guide_mfcc != "silence" else self.engine.silence_mfcc(aud_feat.shape[1], B)
        else:                             # time-major [B,M,64] like aud_feat -> [B,64,M]
            gmc = None if guide_mfcc is None else guide_mfcc.transpose(1, 2).contiguous()
        guide = guide_kwargs(guidance, gmc, guide_id, guide_style, keep_logp, self.engine, B, aud_feat.shape[1])
        noise = self._draw_noise(T, B, noise_fn, temperature, top_k, top_p, min_p, seeds)
        ctl = sample_controls(temperature, top_k, keep_logp, top_p, min_p)
        ctl.update(shaping)
        if noise is None and seeds is not None and sampled(temperature):
            ctl["seeds"] = seeds
        if anchors is not None:
            ctl["anchors"] = anchors
        if style is not None:
            ctl["style"] = style
        if guide:
            gm = guide.pop("guide_mfcc")                   # [B,64,M] or None
            ga = None if gm is None else self.engine.audio_encode(gm)
            if pre_latents is not None:
                gpa = pre_audio if guide_pre_audio is None else guide_pre_audio
                gpa = gpa[..., 0] if gpa.dim() == 4 else gpa
                ga = torch.cat([gpa.to(a.device), a if ga is None else ga], 2)
            guide["guide_aud"] = ga
            ctl.update(guide)
        if pre_latents is None:
            out = self.engine.pixelcnn_generate(a, label, noise, **ctl)
        else:
            pa = pre_audio[..., 0] if pre_audio.dim() == 4 else pre_audio              # [B,256,T0]
            out = self.engine.pixelcnn_generate(torch.cat([pa.to(a.device), a], 2), label, noise, T=T,
                                                pre_latents=pre_latents, **ctl)
        latents = out[0] if (keep_logp or guide) and isinstance(out, tuple) else out
        self.last_logp = out[1] if keep_logp else None
        self.last_kept = out[2] if ctl.get("want_kept") else None
        self.last_guide_logp = out[-1] if guide and keep_logp else None
        body = self.engine.vq_decode(0, latents[..., 0].contiguous())
        hand = self.engine.vq_decode(1, latents[..., 1].contiguous())
        return latents, a.unsqueeze(-1).repeat(1, 1, 1, 2), body, hand

    def _infer_continuity(self, aud_fn, id, fps, sr, B, keep_logp=False, style=None, **ctl):
        """continuity=True (:244-269): a 2 s prefix, then the rest conditioned on the prefix's latents and audio.  The two
        chunks go through the audio encoder separately and are DECODED separately, so each chunk sees zero padding at the
        2 s seam.  ``style`` covers the whole clip (rows T_a + T_b): chunk 0 gets rows [0, T_a), chunk 1, whose prefix is
        chunk 0, all of them.  Per-clip controls apply to both chunks of their clip."""
        aud_feat, gap = get_mfcc_sepa(aud_fn, sr=sr, fps=fps)                 # (M0+M1, 64), M0
        feat = torch.from_numpy(np.ascontiguousarray(np.asarray(aud_feat, dtype=np.float32)))[None].repeat(B, 1, 1)   # [B,M,64]
        label = torch.tensor([0]) if id is None else id.reshape(-1).repeat(B)
        st0 = st1 = None
        if style is not None:
            ta = self.engine.latent_rows(gap)
            st1 = check_style(style, B, ta + self.engine.latent_rows(feat.shape[1] - gap), self.engine.pixelcnn_ncls)
            st0 = st1[:, :ta]
        pre_pose = {"b": None, "h": None}
        lat0, audio0, body_0, hand_0 = self.infer(feat[:, :gap], 0, label, B, pre_pose=pre_pose, keep_logp=keep_logp,
                                                  style=st0, **ctl)
        logp0, kept0 = self.last_logp, self.last_kept
        pre_pose["b"], pre_pose["h"] = body_0[:, :, -4:].transpose(1, 2), hand_0[:, :, -4:].transpose(1, 2)
        lat1, _, body_1, hand_1 = self.infer(feat[:, gap:], 0, label, B, lat0, audio0, pre_pose, keep_logp=keep_logp,
                                             style=st1, **ctl)
        self.last_codes = torch.cat([lat0, lat1], 1)
        self.last_logp = torch.cat([logp0, self.last_logp], 1) if keep_logp else None
        self.last_kept = torch.cat([kept0, self.last_kept], 1) if kept0 is not None else None
        body, hand = torch.cat([body_0, body_1], 2), torch.cat([hand_0, hand_1], 2)
        return torch.cat([body, hand], 1).transpose(1, 2).cpu().numpy()
