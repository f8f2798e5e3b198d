"""Oracle of per-clip sampling controls (ts_pixelcnn_sample_clips / ts_body_sample_clips, include/talkshow_b200.h): the
existing draw of oracle_nucleus.draw applied to each clip with that clip's (temperature, top_k, top_p, min_p), on the
logits of the styled / anchored sampler of oracle_style.  No draw arithmetic of its own."""
import torch

import oracle_anchored as OA
import oracle_nucleus as ON
import oracle_sampling as OSM
import oracle_style as OST
import talkshow_oracle as O


def settings_of(clip):
    """A ``CLIP_CTL`` array (talkshow_b200.engine) or a sequence of 4-tuples -> list of (temperature, top_k, top_p,
    min_p) as the fp32 values the engine receives, as Python numbers."""
    if hasattr(clip, "dtype") and clip.dtype.names:
        return [(float(c["temperature"]), int(c["top_k"]), float(c["top_p"]), float(c["min_p"])) for c in clip]
    return [(float(torch.tensor(t, dtype=torch.float32)), int(k), float(torch.tensor(p, dtype=torch.float32)),
             float(torch.tensor(m, dtype=torch.float32))) for t, k, p, m in clip]


def pixelcnn_sample(sd, style, T, B, aud_feat, noise, clip, anchors=None, pre_latents=None, pre_audio=None, window=18):
    """oracle_style.pixelcnn_sample where clip b draws with clip[b] = (temperature, top_k, top_p, min_p) ->
    (codes [B,T,2], logp [B,T,2], kept [B,T,2] int32)."""
    clip = settings_of(clip)
    assert len(clip) == B
    x = torch.zeros((B, T, 2), dtype=torch.int64)
    h0 = 0
    if pre_latents is not None:
        x = torch.cat([pre_latents, x], 1)
        aud_feat = torch.cat([pre_audio, aud_feat], 2)
        h0 = pre_latents.shape[1]
    pin = torch.zeros(B, T, 2, dtype=torch.bool) if anchors is None else OA.pinned(anchors)
    logp = torch.zeros(B, T, 2)
    kept = torch.zeros(B, T, 2, dtype=torch.int32)
    step = 0
    for i in range(h0, h0 + T):
        lo = 0 if window is None else max(0, i - window + 1)
        for j in range(2):
            lg = OST.pixelcnn_forward(sd, x[:, lo:i + 1], style[:, lo:i + 1], aud_feat[:, :, lo:i + 1])[:, :, i - lo, j]
            for b, (t, k, p, m) in enumerate(clip):
                q = None if (noise is None or t == 0) else noise[step][b:b + 1]
                code, kn = ON.draw(lg[b:b + 1], q, t, k, p, m)
                if pin[b, i - h0, j]:
                    code, kn = anchors[b:b + 1, i - h0, j], torch.zeros(1, dtype=torch.int32)
                x[b, i, j] = code[0]
                kept[b, i - h0, j] = kn[0]
            logp[:, i - h0, j] = OSM.logp_of(lg, x[:, i, j])
            step += 1
    return x[:, h0:], logp, kept


def body_sample(ckpt, vq_ckpt, mfcc, style, noise, clip, anchors=None, window=18):
    """-> (codes, poses [B,4T,C], logp, kept) of the per-clip body call"""
    B = mfcc.shape[0]
    audio = O.audio_encoder(ckpt["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
    lat, logp, kept = pixelcnn_sample(ckpt["generator"], style, audio.shape[2], B, audio, noise, clip, anchors=anchors,
                                      window=window)
    body = O.vq_decode(vq_ckpt["g_body"], lat[..., 0])
    hand = O.vq_decode(vq_ckpt["g_hand"], lat[..., 1])
    return lat, torch.cat([body, hand], 1).transpose(1, 2), logp, kept
