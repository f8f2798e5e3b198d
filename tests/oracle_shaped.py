"""Oracle of logit shaping (ts_pixelcnn_sample_shaped / ts_body_sample_shaped, include/talkshow_b200.h): a repetition
penalty over each clip's recent codes of the draw's column, then an additive code bias, applied to the raw logits before
the existing per-clip draw of oracle_clip_ctl (oracle_nucleus.draw).  A code whose shaped logit is -inf is never drawn
and is not counted in the keep set; log p stays that of the raw prior.  Also the oracle-backed CPU engine of the host
tests, with the shaped draw."""
import numpy as np
import torch

import oracle_anchored as OA
import oracle_clip_ctl as OCC
import oracle_nucleus as ON
import oracle_sampling as OSM
import oracle_style as OST
import talkshow_oracle as O
from oracle_engine import OracleEngine


def penalise(l, history, theta):
    """l [2048] fp32 with every code of ``history`` (each once) divided by theta where positive, multiplied by it
    otherwise (IEEE fp32, as the engine)."""
    if theta == 1.0 or history.numel() == 0:
        return l
    l = l.clone()
    idx = torch.unique(history)
    v = l[idx]
    l[idx] = torch.where(v > 0, v / theta, v * theta)
    return l


def shape(l, history, theta, bias_row=None):
    """The shaped logits of one draw: the penalty over ``history`` (the clip's codes at the draw's column in the window),
    then the bias row (fp32 add)."""
    l = penalise(l, history, float(np.float32(theta)))
    return l if bias_row is None else l + bias_row


def draw(shaped, noise, temperature, top_k=0, top_p=1.0, min_p=0.0):
    """One draw over shaped logits [n,2048] -> (code [n], kept [n] int32).  The code is oracle_nucleus.draw's (a -inf logit
    has probability 0 under every control); the keep set leaves out the -inf codes."""
    code, kept = ON.draw(shaped, noise, temperature, top_k, top_p, min_p)
    if temperature == 0:
        return code, kept
    if top_p < 1.0 or min_p > 0.0:
        keep = ON.keep_mask(shaped, temperature, top_k, top_p, min_p)
    else:
        keep = OSM.keep_mask(shaped, top_k)
    return code, (keep & (shaped != float("-inf"))).sum(-1).to(torch.int32)


def shape_settings(shape_arr):
    """A ``CLIP_SHAPE`` array (talkshow_b200.engine) or a sequence of (theta, W) -> list of (theta as fp32, W)."""
    if hasattr(shape_arr, "dtype") and shape_arr.dtype.names:
        return [(float(s["repetition_penalty"]), int(s["repetition_window"])) for s in shape_arr]
    return [(float(np.float32(t)), int(w)) for t, w in shape_arr]


def pixelcnn_sample(sd, style, T, B, aud_feat, noise, clip, shapes, bias=None, anchors=None, pre_latents=None, pre_audio=None,
                    window=18, return_logits=False):
    """oracle_clip_ctl.pixelcnn_sample with each sampled draw shaped by clip b's (theta, W) = shapes[b] and bias [B,2,2048]
    (or None) -> (codes [B,T,2], logp [B,T,2], kept [B,T,2] int32 (, raw logits [2T,B,2048]))."""
    clip, shapes = OCC.settings_of(clip), shape_settings(shapes)
    assert len(clip) == B and len(shapes) == B
    x = torch.zeros((B, T, 2), dtype=torch.int64)
    h0 = 0
    if pre_latents is not None:
        x = torch.cat([pre_latents, x], 1)
        aud_feat = torch.cat([pre_audio, aud_feat], 2)
        h0 = pre_latents.shape[1]
    pin = torch.zeros(B, T, 2, dtype=torch.bool) if anchors is None else OA.pinned(anchors)
    logp = torch.zeros(B, T, 2)
    kept = torch.zeros(B, T, 2, dtype=torch.int32)
    logs = []
    step = 0
    for i in range(h0, h0 + T):
        lo = 0 if window is None else max(0, i - window + 1)
        for j in range(2):
            lg = OST.pixelcnn_forward(sd, x[:, lo:i + 1], style[:, lo:i + 1], aud_feat[:, :, lo:i + 1])[:, :, i - lo, j]
            if return_logits:
                logs.append(lg.clone())
            for b, ((t, k, p, m), (theta, W)) in enumerate(zip(clip, shapes)):
                if pin[b, i - h0, j]:
                    code, kn = anchors[b:b + 1, i - h0, j], torch.zeros(1, dtype=torch.int32)
                else:
                    s = shape(lg[b], x[b, max(0, i - W):i, j], theta, None if bias is None else bias[b, j])
                    q = None if (noise is None or t == 0) else noise[step][b:b + 1]
                    code, kn = draw(s[None], q, t, k, p, m)
                x[b, i, j] = code[0]
                kept[b, i - h0, j] = kn[0]
            logp[:, i - h0, j] = OSM.logp_of(lg, x[:, i, j])
            step += 1
    out = (x[:, h0:], logp, kept)
    return out + (torch.stack(logs, 0),) if return_logits else out


def body_sample(ckpt, vq_ckpt, mfcc, style, noise, clip, shapes, bias=None, anchors=None, window=18):
    """-> (codes, poses [B,4T,C], logp, kept) of the shaped body call"""
    B = mfcc.shape[0]
    audio = O.audio_encoder(ckpt["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
    lat, logp, kept = pixelcnn_sample(ckpt["generator"], style, audio.shape[2], B, audio, noise, clip, shapes, bias=bias,
                                      anchors=anchors, window=window)
    body = O.vq_decode(vq_ckpt["g_body"], lat[..., 0])
    hand = O.vq_decode(vq_ckpt["g_hand"], lat[..., 1])
    return lat, torch.cat([body, hand], 1).transpose(1, 2), logp, kept


class ShapedOracleEngine(OracleEngine):
    """OracleEngine whose sampling calls take the controls (scalar or per clip), ``anchors=``, ``style=`` and the shaping
    keywords of Engine and are answered by the shaped draw above.  Every call is recorded in ``calls`` as (method,
    CLIP_CTL array, CLIP_SHAPE array, code bias [B,2,2048] or None)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    def load_pixelcnn(self, sd):
        super().load_pixelcnn(sd)
        self.pixelcnn_ncls = sd["layers.0.class_cond_embedding.weight"].shape[0]

    def _prep(self, name, B, H, label, style, temperature, top_k, top_p, min_p, noise, penalty, window, code_bias):
        from talkshow_b200.engine import check_clip_controls, check_clip_shape, check_code_bias, check_style

        clip = check_clip_controls(temperature, top_k, top_p, min_p, B)
        shapes = check_clip_shape(penalty, window, B)
        bias = None if code_bias is None else check_code_bias(code_bias, B)
        self.calls.append((name, clip, shapes, bias))
        if style is not None:
            st = check_style(style, B, H, self.pixelcnn_ncls)
        else:
            label = label.reshape(-1).to(torch.int64)
            st = OST.onehot(label.expand(B) if label.numel() == 1 else label, self.pixelcnn_ncls, H)
        assert noise is not None or not (clip["temperature"] > 0).any()
        return clip, shapes, bias, st

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, temperature=1.0, top_k=0,
                          want_logp=False, top_p=1.0, min_p=0.0, want_kept=False, anchors=None, style=None,
                          repetition_penalty=1.0, repetition_window=8, code_bias=None):
        B = aud.shape[0]
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        T = aud.shape[2] - T0 if T is None else T
        clip, shapes, bias, st = self._prep("pixelcnn_generate", B, T0 + T, label, style, temperature, top_k, top_p, min_p,
                                            noise, repetition_penalty, repetition_window, code_bias)
        a2 = aud.float().unsqueeze(-1).repeat(1, 1, 1, 2)
        pre = dict(pre_latents=pre_latents, pre_audio=a2[:, :, :T0]) if T0 else {}
        codes, logp, kept = pixelcnn_sample(self.sd["pixelcnn"], st, T, B, a2[:, :, T0:], noise, clip, shapes, bias=bias,
                                            anchors=anchors, window=self.window, **pre)
        out = (codes,) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())
        return out if len(out) > 1 else codes

    def body_generate(self, mfcc, label, noise, want_codes=True, temperature=1.0, top_k=0, want_logp=False, top_p=1.0,
                      min_p=0.0, want_kept=False, anchors=None, style=None, repetition_penalty=1.0, repetition_window=8,
                      code_bias=None):
        B, T = mfcc.shape[0], self.latent_rows(mfcc.shape[2])
        clip, shapes, bias, st = self._prep("body_generate", B, T, label, style, temperature, top_k, top_p, min_p, noise,
                                            repetition_penalty, repetition_window, code_bias)
        codes, poses, logp, kept = body_sample({"generator": self.sd["pixelcnn"], "audioencoder": self.sd["audioenc"]},
                                               {"g_body": self.sd["vq0"], "g_hand": self.sd["vq1"]}, mfcc.float(), st, noise,
                                               clip, shapes, bias=bias, anchors=anchors, window=self.window)
        return ((codes if want_codes else None), poses) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())
