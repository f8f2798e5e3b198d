"""Oracle of the sampler's controls (ts_pixelcnn_sample / ts_body_sample, include/talkshow_b200.h), on top of the
unchanged oracle/talkshow_oracle.py: the reference's generate loop with the controlled draw in place of
``multinomial(softmax(logits))``, and the log-likelihood of each draw under the untempered prior."""
import torch
import torch.nn.functional as F

import talkshow_oracle as O


def keep_mask(logits, top_k):
    """[.., 2048] bool: code kept by top-k (TopKLogitsWarper: logits >= the k-th largest, ties kept); all when off."""
    if not 0 < top_k < logits.shape[-1]:
        return torch.ones_like(logits, dtype=torch.bool)
    return logits >= torch.topk(logits, top_k, -1).values[..., -1:]


def draw(logits, noise, temperature, top_k):
    """One controlled draw per row of logits [n, 2048] with Exp(1) noise [n, 2048] (None for greedy)."""
    if temperature == 0:
        return torch.argmax(logits, -1)                    # first index of the maximum
    keep = keep_mask(logits, top_k)
    s = (logits / temperature).masked_fill(~keep, float("-inf"))
    v = (F.softmax(s, -1) / noise).masked_fill(~keep, float("-inf"))   # a dropped code is never drawn
    code = torch.argmax(v, -1)
    # a temperature so small that logits / temperature overflows leaves every kept p / q NaN: the greedy code (the limit
    # of the tempered draw as the temperature goes to 0)
    lost = (torch.isnan(v) | ~keep).all(-1)
    if lost.any():
        code[lost] = torch.argmax(logits[lost], -1)
    return code


def logp_of(logits, code):
    """log_softmax of the untempered, untruncated logits at the drawn code."""
    return torch.log_softmax(logits, -1).gather(-1, code.unsqueeze(-1)).squeeze(-1)


def pixelcnn_sample(sd, label, T, B, aud_feat, noise, temperature=1.0, top_k=0, pre_latents=None, pre_audio=None,
                    window=18, return_logits=False):
    """talkshow_oracle.pixelcnn_generate with the controlled draw -> (codes [B,T,2], logp [B,T,2] (, logits [2T,B,2048]))."""
    x = torch.zeros((B, T, 2), dtype=torch.int64)
    h0 = 0
    if pre_latents is not None:
        x = torch.cat([pre_latents, x], 1)
        aud_feat = torch.cat([pre_audio, aud_feat], 2)
        h0 = pre_latents.shape[1]
    logp = torch.zeros(B, T, 2)
    logs = []
    step = 0
    for i in range(h0, h0 + T):
        lo = 0 if window is None else max(0, i - window + 1)
        for j in range(2):
            lg = O.pixelcnn_forward(sd, x[:, lo:i + 1], label, aud_feat[:, :, lo:i + 1])[:, :, i - lo, j]
            if return_logits:
                logs.append(lg.clone())
            code = draw(lg, None if noise is None else noise[step], temperature, top_k)
            x[:, i, j] = code
            logp[:, i - h0, j] = logp_of(lg, code)
            step += 1
    out = (x[:, h0:], logp)
    return out + (torch.stack(logs, 0),) if return_logits else out


def body_sample(ckpt, vq_ckpt, mfcc, label, noise, temperature=1.0, top_k=0, window=18):
    """talkshow_oracle.body_generate with the controlled draw -> (codes [B,T,2], poses [B,4T,C], logp [B,T,2])."""
    B = mfcc.shape[0]
    audio = O.audio_encoder(ckpt["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
    lat, logp = pixelcnn_sample(ckpt["generator"], label, audio.shape[2], B, audio, noise, temperature, top_k,
                                window=window)
    body = O.vq_decode(vq_ckpt["g_body"], lat[..., 0])
    hand = O.vq_decode(vq_ckpt["g_hand"], lat[..., 1])
    return lat, torch.cat([body, hand], 1).transpose(1, 2), logp


def reference_noise(seed, steps, B):
    """The Exp(1) draws the reference's multinomial consumes under torch.manual_seed(seed) on the CPU: one
    ``exponential_`` of [B,2048] per sampled position."""
    torch.manual_seed(seed)
    out = torch.empty(steps, B, 2048)
    for s in range(steps):
        out[s] = torch.empty(B, 2048).exponential_(1)
    return out
