"""Oracle of guided sampling (ts_pixelcnn_sample_guided / ts_body_sample_guided, include/talkshow_b200.h): for pair p,
g = l_c + s (l_c - l_u) with s = w_p - 1, each operation rounded to fp32 on its own, then the shaped draw of
oracle_shaped (the pair's penalty over its history and bias, then its controls).  Both branches take the drawn code;
each branch's log p is that of its own raw logits."""
import numpy as np
import torch

import oracle_sampling as OSM
import oracle_shaped as OSH
import oracle_style as OST


def guided_logits(lc, lu, w):
    """g = lc + (w - 1) (lc - lu) [.., 2048] in fp32: subtract, multiply, add, each rounded (numpy float32, no FMA)."""
    lc = np.asarray(lc, np.float32)
    lu = np.asarray(lu, np.float32)
    s = np.float32(np.float32(w) - np.float32(1.0))
    g = np.float32(lc + np.float32(s * np.float32(lc - lu)))
    return torch.from_numpy(np.asarray(g, np.float32).copy())


def draw(lc, lu, w, noise, temperature, top_k=0, top_p=1.0, min_p=0.0, history=None, theta=1.0, bias_row=None):
    """One guided draw of one pair: raw logits lc, lu [2048], noise [2048] (or None when greedy) -> (code, kept)."""
    g = guided_logits(lc, lu, w)
    if history is not None or bias_row is not None:
        g = OSH.shape(g, torch.zeros(0, dtype=torch.int64) if history is None else history, theta, bias_row)
    code, kept = OSH.draw(g[None], None if noise is None else noise[None], temperature, top_k, top_p, min_p)
    return int(code[0]), int(kept[0])


def pixelcnn_sample(sd, style2, T, P, aud2, noise, clip, shapes, guidance, bias=None, pre_latents=None, pre_audio2=None,
                    window=18):
    """The guided call on the CPU: style2 [2P,T0+T,ncls] and aud2 [2P,256,T,2] per branch (2p the clip, 2p + 1 its
    negative conditioning), noise [2T,P,2048], clip / shapes / guidance / bias per pair, pre_latents [P,T0,2] (fed to both
    branches) with pre_audio2 [2P,256,T0,2] -> (codes [2P,T,2], logp [2P,T,2], kept [2P,T,2])."""
    clip, shapes = OSH.OCC.settings_of(clip), OSH.shape_settings(shapes)
    x = torch.zeros((2 * P, T, 2), dtype=torch.int64)
    h0 = 0
    if pre_latents is not None:
        x = torch.cat([pre_latents.repeat_interleave(2, 0), x], 1)
        aud2 = torch.cat([pre_audio2, aud2], 2)
        h0 = pre_latents.shape[1]
    logp = torch.zeros(2 * P, T, 2)
    kept = torch.zeros(2 * P, T, 2, dtype=torch.int32)
    step = 0
    for i in range(h0, h0 + T):
        lo = 0 if window is None else max(0, i - window + 1)
        for j in range(2):
            lg = OST.pixelcnn_forward(sd, x[:, lo:i + 1], style2[:, lo:i + 1], aud2[:, :, lo:i + 1])[:, :, i - lo, j]
            for p, ((t, k, tp, mp), (theta, W)) in enumerate(zip(clip, shapes)):
                q = None if (noise is None or t == 0) else noise[step][p]
                code, kn = draw(lg[2 * p], lg[2 * p + 1], float(guidance[p]), q, t, k, tp, mp,
                                history=x[2 * p, max(0, i - W):i, j], theta=theta,
                                bias_row=None if bias is None else bias[p, j])
                x[2 * p:2 * p + 2, i, j] = code
                kept[2 * p:2 * p + 2, i - h0, j] = kn
            logp[:, i - h0, j] = OSM.logp_of(lg, x[:, i, j])
            step += 1
    return x[:, h0:], logp, kept
