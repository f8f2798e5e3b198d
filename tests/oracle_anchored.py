"""Oracle of anchored sampling (ts_pixelcnn_sample_anchored / ts_body_sample_anchored, include/talkshow_b200.h), on top of
oracle_nucleus.py.  The rule: anchors [B,T,2] over the sampled rows; a value in [0, 2048) pins the draw to that code (no
draw, its noise unused, log p = log_softmax of its untempered logits at the anchor, keep-set size 0), any other value
samples the draw as the call without anchors would.  The prior is causal, so a pinned code conditions later draws only."""
import torch

import oracle_nucleus as ON
import oracle_sampling as OSM
import talkshow_oracle as O

NCODE = 2048


def pinned(anchors):
    """[..] bool: the draws an anchors tensor pins"""
    return (anchors >= 0) & (anchors < NCODE)


def pixelcnn_sample(sd, label, T, B, aud_feat, noise, anchors, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0,
                    pre_latents=None, pre_audio=None, window=18):
    """oracle_nucleus.pixelcnn_sample with anchors [B,T,2] -> (codes [B,T,2], logp [B,T,2], kept [B,T,2] int32, margins
    [B,T,2,2] float64; a pinned draw has margin inf: it has no keep set that could change)."""
    x = torch.zeros((B, T, 2), dtype=torch.int64)
    h0 = 0
    if pre_latents is not None:
        x = torch.cat([pre_latents, x], 1)
        aud_feat = torch.cat([pre_audio, aud_feat], 2)
        h0 = pre_latents.shape[1]
    pin = pinned(anchors)
    logp = torch.zeros(B, T, 2)
    kept = torch.zeros(B, T, 2, dtype=torch.int32)
    margin = torch.full((B, T, 2, 2), float("inf"), dtype=torch.float64)
    step = 0
    for i in range(h0, h0 + T):
        lo = 0 if window is None else max(0, i - window + 1)
        for j in range(2):
            lg = O.pixelcnn_forward(sd, x[:, lo:i + 1], label, aud_feat[:, :, lo:i + 1])[:, :, i - lo, j]
            p = pin[:, i - h0, j]
            code, kn = ON.draw(lg, None if noise is None else noise[step], temperature, top_k, top_p, min_p)
            if temperature > 0 and (top_p < 1.0 or min_p > 0.0):
                _, mp, mm = ON.keep_mask(lg, temperature, top_k, top_p, min_p, return_margin=True)
                margin[:, i - h0, j, 0] = torch.where(p, float("inf"), mp)
                margin[:, i - h0, j, 1] = torch.where(p, float("inf"), mm)
            code = torch.where(p, anchors[:, i - h0, j], code)
            x[:, i, j] = code
            kept[:, i - h0, j] = torch.where(p, 0, kn)
            logp[:, i - h0, j] = OSM.logp_of(lg, code)
            step += 1
    return x[:, h0:], logp, kept, margin


def body_sample(ckpt, vq_ckpt, mfcc, label, noise, anchors, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, window=18):
    """-> (codes, poses [B,4T,C], logp, kept, margins) of the anchored body call."""
    B = mfcc.shape[0]
    audio = O.audio_encoder(ckpt["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
    lat, logp, kept, margin = pixelcnn_sample(ckpt["generator"], label, audio.shape[2], B, audio, noise, anchors, temperature,
                                              top_k, top_p, min_p, window=window)
    body = O.vq_decode(vq_ckpt["g_body"], lat[..., 0])
    hand = O.vq_decode(vq_ckpt["g_hand"], lat[..., 1])
    return lat, torch.cat([body, hand], 1).transpose(1, 2), logp, kept, margin


def teacher_forced_draw(sd, codes, label, aud, noise, anchors):
    """The default draw (temperature 1) of every position on the teacher-forced logits of ``codes`` [B,T,2], with the
    pinned draws replaced by their anchors: equals ``codes`` when they are the anchored sampler's output for ``noise``."""
    B, T = codes.shape[:2]
    logits = O.pixelcnn_forward(sd, codes, label, aud.unsqueeze(-1).repeat(1, 1, 1, 2))          # [B,2048,T,2]
    lg = logits.permute(2, 3, 0, 1).reshape(2 * T * B, NCODE)
    ref = OSM.draw(lg, noise.reshape(2 * T * B, NCODE), 1.0, 0).reshape(T, 2, B).permute(2, 0, 1)
    return torch.where(pinned(anchors), anchors, ref)
