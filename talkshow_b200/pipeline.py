"""Whole-body batch generation (what scripts/demo.py:158-229 does per clip, batched) and its
multi-GPU sharding.

A batch of clips / diversity samples is a set of independent autoregressive chains (SURVEY.md §8e):
rank r of G takes a contiguous slice of the batch, runs face + body + pose assembly on its own
GPU, and ONE NCCL all-gather of the final [b,F,265] pose tensor rebuilds the batch on every rank.
No other collective is on the path.
"""
from __future__ import annotations

import torch

from .engine import (Engine, check_anchors, check_clip_controls, check_clip_shape, check_code_bias, check_guidance, check_style,
                     guide_kwargs, per_clip, resolve_clip_seeds, sample_controls, sampled, shaping_kwargs)
from .nets.base import draw_sampler_noise


def shard_range(B, rank, world):
    """Contiguous slice of the batch owned by ``rank`` (first B % world ranks get one extra)."""
    base, rem = divmod(B, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class WholeBody:
    """face (jaw+expression) + body/hands + part2full assembly -> SMPL-X parameters [B,F,265].

    ``overlap_batch`` > 0: batches up to that size run the body path and the face path SIDE BY SIDE on two streams.  The
    sampler is a serial chain of 3 900 stages that is latency-bound at every batch size (it loses little time on fewer
    SMs), so a second engine holds a sampler plan for ``overlap_ctas`` persistent CTAs launched as CTA pairs (whole TPCs,
    high-priority stream) and the face kernels fill the remaining TPCs, then the whole GPU.  Results are bit-identical to the
    sequential order (same kernels, same arithmetic; tests/test_gpu_baseline_shapes.py)."""

    def __init__(self, engine: Engine, overlap_batch=64, overlap_ctas=96):
        self.e = engine
        self.device = engine.device
        self.overlap_batch = overlap_batch if not getattr(engine, "host_only", True) else 0
        self.overlap_ctas = overlap_ctas
        self.e2 = None            # body path engine with the partial-GPU sampler plan (same device)
        self._side = None
        self._body_engine = engine   # the engine whose sampler ran in the last generate()

    def load(self, pixel_ckpt, vq_ckpt, face_ckpt):
        """Checkpoint dicts in the reference's formats (talkshow_b200/synth.py docstring)."""
        self.e.load_pixelcnn(pixel_ckpt["generator"])
        self.e.load_audioenc(pixel_ckpt["audioencoder"])
        self.e.load_vq(0, vq_ckpt["g_body"])
        self.e.load_vq(1, vq_ckpt["g_hand"])
        self.e.load_face(face_ckpt["generator"])
        dim = pixel_ckpt["generator"]["embedding.weight"].shape[1]
        if self.overlap_batch > 0 and dim == 256 and self.overlap_ctas < self.e.sm_count:
            idx = self.device.index or 0
            self.e2 = Engine(idx)
            self.e2.set_pixelcnn_ctas(self.overlap_ctas)
            self.e2.load_pixelcnn(pixel_ckpt["generator"])
            self.e2.load_audioenc(pixel_ckpt["audioencoder"])
            self.e2.load_vq(0, vq_ckpt["g_body"])
            self.e2.load_vq(1, vq_ckpt["g_hand"])
            self._side = torch.cuda.Stream(device=self.device, priority=-1)   # the sampler CTAs are placed before queued face CTAs

    @property
    def launches(self):
        """Kernels launched by the library so far (both engines)."""
        return self.e.launches + (self.e2.launches if self.e2 is not None else 0)

    def pixelcnn_timing(self, enable=True):
        self.e.pixelcnn_timing(enable)
        if self.e2 is not None:
            self.e2.pixelcnn_timing(enable)

    def pixelcnn_last_ms(self):
        """Device time of the sampler launch of the last ``generate`` (events on its launch stream, inside the library)."""
        return self._body_engine.pixelcnn_last_ms()

    def close(self):
        if self.e2 is not None:
            torch.cuda.synchronize(self.device)
            self.e2.close()
            self.e2 = None

    def generate(self, mfcc, wave, label, noise=None, stand=False, per_step_noise=True, temperature=1.0, top_k=0,
                 keep_logp=False, top_p=1.0, min_p=0.0, clip_seeds=None, anchors=None, keep_codes=False, style=None,
                 repetition_penalty=1.0, repetition_window=8, code_bias=None, guidance=None, guide_mfcc=None, guide_label=None,
                 guide_style=None):
        """mfcc [B,64,M], wave [B,N] (16 kHz), label [B] on the device -> poses [B,F,265] (device).
        F = N*30//16000 face frames; the body (4*T frames) is padded/truncated to F like demo.py:207-211.
        Sampling controls of the body prior as in s2g_body_pixel.generate: ``temperature`` (0 = greedy, no noise is
        drawn), ``top_k``, ``top_p``, ``min_p``; ``keep_logp`` keeps each draw's log-likelihood under the untempered prior
        as self.last_logp [B,T,2] and, with top_p or min_p on, the size of its keep set as self.last_kept [B,T,2].
        ``clip_seeds`` (an integer s: clip b gets s + b; or a length-B sequence / int64 tensor): seeded sampling, no noise
        is drawn and each clip's motion depends only on its seed.  Not combinable with ``noise``.
        ``anchors`` [B,T,2] pins draws of the body prior (s2g_body_pixel.generate: a code pins, -1 samples).
        ``keep_codes`` keeps the body codes of the call, pinned and drawn, as self.last_codes [B,T,2] (None otherwise):
        the codes a later call can anchor to.
        ``style`` [B,T,ncls] or [B,ncls]: a speaker schedule for the body prior (s2g_body_pixel.generate), ``label`` is then
        not read.  The face path keeps the demo's zero id (demo.py:173-181) whatever the style: the body prior is the only
        net styled here (s2g_face.generate_ids takes a soft id for the face).
        ``temperature`` / ``top_k`` / ``top_p`` / ``min_p`` may each be given per clip (s2g_body_pixel.generate): one batch
        serves clips with different settings, on the overlapped and the sequential path alike.
        ``repetition_penalty`` / ``repetition_window`` / ``code_bias``: logit shaping of the body prior
        (s2g_body_pixel.generate), on both paths.
        ``guidance`` with ``guide_mfcc`` ([B,64,M] or "silence"), ``guide_label`` and / or ``guide_style``: guided
        sampling of the body prior (s2g_body_pixel.generate); with ``keep_logp`` the negative branches' log p is kept as
        self.last_guide_logp."""
        B, _, M = mfcc.shape
        frame = wave.shape[1] * 30 // 16000
        T = self.e.latent_rows(M)
        shaping = shaping_kwargs(repetition_penalty, repetition_window, code_bias, B)
        guide = guide_kwargs(guidance, guide_mfcc, guide_label, guide_style, keep_logp, self.e, B, M)
        ctl = sample_controls(temperature, top_k, keep_logp, top_p, min_p)
        ctl.update(shaping)
        ctl.update(guide)
        want_kept = bool(ctl.get("want_kept"))
        if noise is not None and clip_seeds is not None:
            raise ValueError("WholeBody.generate: noise and clip_seeds are two noise sources; give one")
        seeds = resolve_clip_seeds(clip_seeds, B)
        if seeds is not None and sampled(temperature):
            ctl["seeds"] = seeds
        elif noise is None and sampled(temperature):
            noise = draw_sampler_noise(T, B, self.device, per_step=per_step_noise)
        if anchors is not None:
            ctl["anchors"] = anchors
        if style is not None:
            ctl["style"] = style
        idz = torch.zeros(B, 4, device=self.device)                    # demo.py:173-181: id not passed
        if self.e2 is not None and B <= self.overlap_batch:
            # small batch: sampler (on overlap_ctas SMs, launched first) and face regressor (on the free TPCs) side by side
            cur = torch.cuda.current_stream(self.device)
            self._side.wait_stream(cur)
            self._body_engine = self.e2
            with torch.cuda.stream(self._side):
                out = self.e2.body_generate(mfcc, label, noise, want_codes=keep_codes, **ctl)
            body = out[1]
            self.last_codes = out[0]
            self.last_logp = out[2] if keep_logp else None
            self.last_kept = out[3] if want_kept else None
            self.last_guide_logp = out[-1] if guide and keep_logp else None
            face = self.e.face_forward(wave, idz, frame)
            cur.wait_stream(self._side)
            body.record_stream(cur)                                      # allocated on the side stream, consumed here
            if keep_logp:
                self.last_logp.record_stream(cur)
            if want_kept:
                self.last_kept.record_stream(cur)
            if keep_codes:
                self.last_codes.record_stream(cur)
            if self.last_guide_logp is not None:
                self.last_guide_logp.record_stream(cur)
            for t in (mfcc, label, noise, ctl.get("seeds"), ctl.get("anchors"), ctl.get("style"), ctl.get("code_bias"),
                      ctl.get("guide_mfcc"), ctl.get("guide_label"), ctl.get("guide_style")):
                if torch.is_tensor(t) and t.is_cuda:
                    t.record_stream(self._side)                          # allocated here, consumed on the side stream
            return self.e.assemble_pose(face, body, stand)
        self._body_engine = self.e
        face = self.e.face_forward(wave, idz, frame)
        out = self.e.body_generate(mfcc, label, noise, want_codes=keep_codes, **ctl)
        self.last_codes = out[0]
        self.last_logp = out[2] if keep_logp else None
        self.last_kept = out[3] if want_kept else None
        self.last_guide_logp = out[-1] if guide and keep_logp else None
        return self.e.assemble_pose(face, out[1], stand)

    def evaluate(self, bat):
        """Score held-out clips under the loaded face / VQ / prior trio: what s2g_face.evaluate, s2g_body_vq.evaluate and
        s2g_body_pixel.evaluate return, in one call, with the VQ encoder run once (the codes of the VQ score feed the prior
        score).  bat: 'wave' [B,N] (16 kHz, the face input), 'aud_feat' [B,64,M] (MFCC), 'poses' [B,165,F] ([B,330,F] for a
        convert_to_6d trio), 'expression' [B,100,F], 'speaker' [B].  F must be a multiple of 4 and M must give F/4 latent
        rows.  Returns (None, {'MSELoss', 'exp_loss', 'brec_loss', 'bvelocity_loss', 'hrec_loss', 'hvelocity_loss',
        'ce_loss'}); per-clip values are kept as self.last_losses, the per-position prior NLL as self.last_nll."""
        import torch.nn.functional as F

        from .data_utils.lower_body import c_index_3d, c_index_6d
        from .nets.smplx_body_vq import check_pose_block, score_vq_pair
        from .nets.smplx_face import face_gt, score_face

        six = self.e.vq_dim(0) == 78
        poses = torch.as_tensor(bat["poses"]).to(torch.float32)
        check_pose_block(poses, six, "WholeBody.evaluate")
        mfcc = torch.as_tensor(bat["aud_feat"]).to(torch.float32)
        B, nf = poses.shape[0], poses.shape[2]
        if mfcc.dim() != 3 or mfcc.shape[0] != B or self.e.latent_rows(mfcc.shape[2]) != nf // 4:
            # the reference fails in the prior's concatenation of code and audio rows (gated_pixelcnn_v2.py:143)
            raise ValueError("WholeBody.evaluate: aud_feat %s gives %d latent rows, %d pose frames give %d"
                             % (tuple(mfcc.shape), self.e.latent_rows(mfcc.shape[2]) if mfcc.dim() == 3 else -1, nf, nf // 4))
        wave = torch.as_tensor(bat["wave"]).to(torch.float32).reshape(B, -1)
        label = (torch.as_tensor(bat["speaker"]) - 20).reshape(-1).to(torch.int64)
        face_losses, face_clip = score_face(self.e, wave, F.one_hot(label, 4).to(torch.float32),
                                            face_gt(poses, torch.as_tensor(bat["expression"])))
        gt = poses[:, c_index_6d if six else c_index_3d, :].permute(0, 2, 1)
        codes, vq_losses, vq_clip = score_vq_pair(self.e, gt, 78 if six else 39)
        nll = self.e.pixelcnn_score(self.e.audio_encode(mfcc), label, codes)
        self.last_nll = nll
        self.last_losses = dict(face_clip, **vq_clip)
        return None, dict(face_losses, **vq_losses, ce_loss=float(nll.double().mean()))

    def generate_sharded(self, mfcc, wave, label, rank, world, noise_full=None, seed=None, stand=False, gather=True,
                         group=None, temperature=1.0, top_k=0, keep_logp=False, top_p=1.0, min_p=0.0, clip_seeds=None,
                         anchors=None, style=None, repetition_penalty=1.0, repetition_window=8, code_bias=None,
                         guidance=None, guide_mfcc=None, guide_label=None, guide_style=None):
        """Multi-GPU form of ``generate`` whose RESULT DOES NOT DEPEND ON ``world`` (SURVEY.md §8e): the arguments are
        the FULL batch (host or device tensors, identical on every rank), the sampler noise is drawn for the full batch in
        the reference's order — ``noise_full`` [2T,B,2048], or drawn here from ``seed`` on this rank's device generator
        (same seed on every rank gives every rank the same stream) — and rank r keeps the slice of its contiguous shard
        ``shard_range(B, r, world)``.  Each rank runs its shard; ONE all-gather rebuilds [B,F,265] everywhere.
        Sampling controls as in ``generate`` (greedy decoding draws no noise); with ``keep_logp`` self.last_logp holds
        this rank's shard (and self.last_kept, as in ``generate``).
        ``clip_seeds`` (as in ``generate``, for the full batch): seeded sampling; rank r passes the seeds of its shard and
        draws no noise at all, and the gathered result equals ``generate`` with the same seeds on one GPU.  ``seed`` keeps
        its meaning (the torch stream of the full-batch noise) and is not used with ``clip_seeds``.
        ``anchors`` [B,T,2] (as in ``generate``, for the full batch): rank r passes the rows of its shard, so the gathered
        result equals ``generate`` with the same anchors on one GPU.  ``style`` [B,T,ncls] or [B,ncls] (full batch, as in
        ``generate``): rank r passes its shard's rows.  Per-clip ``temperature`` / ``top_k`` / ``top_p`` / ``min_p`` (full
        batch, as in ``generate``): rank r passes its shard's values.  ``repetition_penalty`` / ``repetition_window`` (scalar
        or per clip) and ``code_bias`` ([2,2048] or [B,2,2048]) as in ``generate``: rank r passes its shard's values and bias
        rows.  ``guidance`` (scalar or per clip) and the negative conditioning (full batch, as in ``generate``): rank r
        passes its shard's clips, each with its own negative branch, so a pair is never split across ranks."""
        B, _, M = mfcc.shape
        lo, hi = shard_range(B, rank, world)
        T = self.e.latent_rows(M)
        # validated before any noise is drawn; generate() gets the controls only when they differ from the defaults
        sc = sample_controls(temperature, top_k, keep_logp, top_p, min_p)
        ctl = dict(temperature=temperature, top_k=top_k, keep_logp=keep_logp) if sc else {}
        if "top_p" in sc:
            ctl.update(top_p=top_p, min_p=min_p)
        if per_clip(temperature, top_k, top_p, min_p):
            cc = check_clip_controls(temperature, top_k, top_p, min_p, B)[lo:hi]
            ctl.update(temperature=cc["temperature"], top_k=cc["top_k"], top_p=cc["top_p"], min_p=cc["min_p"])
        if noise_full is not None and clip_seeds is not None:
            raise ValueError("WholeBody.generate_sharded: noise_full and clip_seeds are two noise sources; give one")
        seeds = resolve_clip_seeds(clip_seeds, B)
        if anchors is not None:
            ctl["anchors"] = check_anchors(anchors, B, T)[lo:hi]
        if style is not None:
            ctl["style"] = check_style(style, B, T, self.e.pixelcnn_ncls)[lo:hi]
        if shaping_kwargs(repetition_penalty, repetition_window, code_bias, B):
            shape = check_clip_shape(repetition_penalty, repetition_window, B)[lo:hi]
            ctl.update(repetition_penalty=shape["repetition_penalty"], repetition_window=shape["repetition_window"])
            if code_bias is not None:
                ctl["code_bias"] = check_code_bias(code_bias, B)[lo:hi]
        if guidance is not None:
            ctl["guidance"] = check_guidance(guidance, B)[lo:hi]
            rows = lambda t: t if t is None or isinstance(t, str) else torch.as_tensor(t)[lo:hi]
            ctl["guide_mfcc"] = rows(guide_mfcc)
            if guide_label is not None:
                gl = torch.as_tensor(guide_label).reshape(-1)
                ctl["guide_label"] = gl.expand(B)[lo:hi] if gl.numel() == 1 else gl[lo:hi]
            if guide_style is not None:
                ctl["guide_style"] = check_style(guide_style, B, T, self.e.pixelcnn_ncls)[lo:hi]
        else:
            guide_kwargs(guidance, guide_mfcc, guide_label, guide_style)   # a negative conditioning alone raises
        if seeds is not None:
            ctl["clip_seeds"] = seeds[lo:hi]
        elif noise_full is None and sampled(temperature):
            g = None
            if seed is not None:
                g = torch.Generator(device=self.device)
                g.manual_seed(int(seed))
            noise_full = draw_sampler_noise(T, B, self.device, generator=g)
        if hi == lo:                                                     # more ranks than samples: nothing to run here
            frame = wave.shape[1] * 30 // 16000
            local = torch.empty(0, frame, 265, device=self.device)
            self.last_logp = torch.empty(0, T, 2, device=self.device) if keep_logp else None
            self.last_kept = torch.empty(0, T, 2, dtype=torch.int32, device=self.device) if sc.get("want_kept") else None
            self.last_guide_logp = (torch.empty(0, T, 2, device=self.device) if guidance is not None and keep_logp
                                    else None)
        else:
            dev = lambda t: t[lo:hi].to(self.device, non_blocking=True)
            nz = None if noise_full is None else noise_full[:, lo:hi].to(self.device).contiguous()
            local = self.generate(dev(mfcc), dev(wave), dev(label), noise=nz, stand=stand, **ctl)
        return allgather_poses(local, B, world, group=group, engine=self.e) if gather else local

    def generate_host(self, mfcc_host, wave_host, label_host, out_host=None, **kw):
        """Public end-to-end call with HOST buffers (pinned for async copies): H2D inputs, generate,
        D2H result.  Returns the host tensor [B,F,265]."""
        mfcc = mfcc_host.to(self.device, non_blocking=True)
        wave = wave_host.to(self.device, non_blocking=True)
        label = label_host.to(self.device, non_blocking=True)
        poses = self.generate(mfcc, wave, label, **kw)
        if out_host is None:
            out_host = torch.empty(poses.shape, dtype=poses.dtype, pin_memory=True)
        out_host.copy_(poses, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return out_host


def allgather_poses(local, B_total, world, group=None, engine=None):
    """ONE all-gather of the pose tensor over NCCL (NVLink/NVSwitch).  local [b,F,265] -> [B_total,F,265].
    Uneven shards are padded to the largest shard for the collective and trimmed afterwards.  With an ``engine`` whose
    communicator was created (``Engine.nccl_init``) the collective is the library's own ``ts_allgather``; otherwise
    torch.distributed's ``all_gather_into_tensor`` (NCCL on GPUs, gloo in the CPU tests)."""
    import torch.distributed as dist

    if world == 1:
        return local
    bmax = -(-B_total // world)
    if local.shape[0] < bmax:
        pad = torch.zeros((bmax - local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        local = torch.cat([local, pad], 0)
    if engine is not None and getattr(engine, "nccl_world", 0) == world:
        out = engine.allgather(local.contiguous())
    else:
        out = torch.empty((world * bmax,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
    if B_total == world * bmax:
        return out
    parts = []
    for r in range(world):
        lo, hi = shard_range(B_total, r, world)
        parts.append(out[r * bmax: r * bmax + (hi - lo)])
    return torch.cat(parts, 0)
