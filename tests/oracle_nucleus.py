"""Oracle of nucleus (top-p) and min-p sampling (ts_pixelcnn_sample_ctl / ts_body_sample_ctl, include/talkshow_b200.h),
on top of oracle_sampling.py: the keep rule on integer masses in int64, the controlled draw over the final keep set, the
size of each keep set and how far each draw's keep set is from changing."""
import numpy as np
import torch
import torch.nn.functional as F

import oracle_sampling as OS
import talkshow_oracle as O


def masses(logits, temperature, top_k=0):
    """e [n,2048] fp32 = exp(l / t - max l / t) over the top-k set (0 elsewhere) and the integer masses w = rint(e 2^32)."""
    keep0 = OS.keep_mask(logits, top_k)
    mx = logits.max(-1, keepdim=True).values
    e = torch.exp(logits / temperature - mx / temperature).masked_fill(~keep0, 0.0)
    w = torch.from_numpy(np.rint(e.numpy().astype(np.float64) * 2.0 ** 32).astype(np.int64))
    return e, w, keep0


def mass_above(logits, w):
    """A [n,2048] int64: the mass of the codes whose logit is strictly greater (ties share one value)."""
    ls, order = torch.sort(logits, dim=-1, descending=True, stable=True)
    ws = w.gather(-1, order)
    excl = torch.cumsum(ws, -1) - ws
    first = torch.ones_like(ls, dtype=torch.bool)
    first[:, 1:] = ls[:, 1:] != ls[:, :-1]
    a_sorted = torch.cummax(torch.where(first, excl, torch.full_like(excl, -1)), -1).values   # excl never decreases
    return torch.empty_like(w).scatter_(-1, order, a_sorted)


def keep_mask(logits, temperature, top_k=0, top_p=1.0, min_p=0.0, return_margin=False):
    """[n,2048] bool: the final keep set of a tempered draw (temperature > 0).  With ``return_margin`` also [n] float64:
    min |A - P| / W over the codes with A > 0 (how far the nucleus is from changing; inf with top_p off) and min |e - m| / m (inf with
    min_p off).  top_p and min_p act as the fp32 values the engine receives."""
    e, w, keep = masses(logits, temperature, top_k)
    n = logits.shape[0]
    m_p = torch.full((n,), float("inf"), dtype=torch.float64)
    m_m = torch.full((n,), float("inf"), dtype=torch.float64)
    if top_p < 1.0:
        A = mass_above(logits, w)
        W = w.sum(-1, keepdim=True).double()
        P = float(np.float32(top_p)) * W                      # one double multiplication, both factors exact
        keep = keep & (A.double() < P)
        # the most likely code has A = 0 in any arithmetic and is always kept: it is no boundary
        m_p = torch.where(A > 0, (A.double() - P).abs() / W, torch.full_like(P, float("inf")).expand_as(A)).min(-1).values
    if min_p > 0.0:
        m = float(np.float32(min_p))
        keep = keep & (e >= m)
        m_m = ((e.double() - m).abs() / m).min(-1).values
    return (keep, m_p, m_m) if return_margin else keep


def draw(logits, noise, temperature, top_k=0, top_p=1.0, min_p=0.0):
    """One draw per row of logits [n,2048] -> (code [n], kept [n] int32).  With top_p and min_p off this is
    oracle_sampling.draw."""
    n = logits.shape[0]
    if temperature == 0:
        return torch.argmax(logits, -1), torch.ones(n, dtype=torch.int32)
    if not (top_p < 1.0 or min_p > 0.0):
        return OS.draw(logits, noise, temperature, top_k), OS.keep_mask(logits, top_k).sum(-1).to(torch.int32)
    keep = keep_mask(logits, temperature, top_k, top_p, min_p)
    s = (logits / temperature).masked_fill(~keep, float("-inf"))
    v = (F.softmax(s, -1) / noise).masked_fill(~keep, float("-inf"))
    code = torch.argmax(v, -1)
    lost = (torch.isnan(v) | ~keep).all(-1)
    if lost.any():
        code[lost] = torch.argmax(logits[lost], -1)
    return code, keep.sum(-1).to(torch.int32)


def pixelcnn_sample(sd, label, T, B, aud_feat, noise, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, pre_latents=None,
                    pre_audio=None, window=18, return_logits=False):
    """oracle_sampling.pixelcnn_sample with top_p / min_p -> (codes [B,T,2], logp [B,T,2], kept [B,T,2] int32, margins
    [B,T,2,2] float64 (nucleus, min-p) (, logits [2T,B,2048]))."""
    x = torch.zeros((B, T, 2), dtype=torch.int64)
    h0 = 0
    if pre_latents is not None:
        x = torch.cat([pre_latents, x], 1)
        aud_feat = torch.cat([pre_audio, aud_feat], 2)
        h0 = pre_latents.shape[1]
    logp = torch.zeros(B, T, 2)
    kept = torch.zeros(B, T, 2, dtype=torch.int32)
    margin = torch.full((B, T, 2, 2), float("inf"), dtype=torch.float64)
    logs = []
    step = 0
    for i in range(h0, h0 + T):
        lo = 0 if window is None else max(0, i - window + 1)
        for j in range(2):
            lg = O.pixelcnn_forward(sd, x[:, lo:i + 1], label, aud_feat[:, :, lo:i + 1])[:, :, i - lo, j]
            if return_logits:
                logs.append(lg.clone())
            code, kn = draw(lg, None if noise is None else noise[step], temperature, top_k, top_p, min_p)
            if temperature > 0 and (top_p < 1.0 or min_p > 0.0):
                _, mp, mm = keep_mask(lg, temperature, top_k, top_p, min_p, return_margin=True)
                margin[:, i - h0, j, 0], margin[:, i - h0, j, 1] = mp, mm
            x[:, i, j] = code
            kept[:, i - h0, j] = kn
            logp[:, i - h0, j] = OS.logp_of(lg, code)
            step += 1
    out = (x[:, h0:], logp, kept, margin)
    return out + (torch.stack(logs, 0),) if return_logits else out


def body_sample(ckpt, vq_ckpt, mfcc, label, noise, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, window=18):
    """oracle_sampling.body_sample with top_p / min_p -> (codes, poses [B,4T,C], logp, kept, margins)."""
    B = mfcc.shape[0]
    audio = O.audio_encoder(ckpt["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
    lat, logp, kept, margin = pixelcnn_sample(ckpt["generator"], label, audio.shape[2], B, audio, noise, temperature, top_k,
                                              top_p, min_p, window=window)
    body = O.vq_decode(vq_ckpt["g_body"], lat[..., 0])
    hand = O.vq_decode(vq_ckpt["g_hand"], lat[..., 1])
    return lat, torch.cat([body, hand], 1).transpose(1, 2), logp, kept, margin


def top_p_reference(logits, temperature, top_p):
    """TopPLogitsWarper in float64 by sort and cumulative sum: keep the smallest prefix of the descending order whose
    probability reaches top_p (a code is kept iff the probability before it is below top_p)."""
    p = torch.softmax(logits.double() / temperature, -1)
    ps, order = torch.sort(p, dim=-1, descending=True, stable=True)
    before = torch.cumsum(ps, -1) - ps
    return torch.zeros_like(p, dtype=torch.bool).scatter_(-1, order, before < float(np.float32(top_p)))
