"""Oracle of styled sampling (ts_pixelcnn_sample_styled / ts_body_sample_styled / ts_pixelcnn_score_styled,
include/talkshow_b200.h), on top of oracle/talkshow_oracle.py and tests/oracle_anchored.py.  The rule: style
[B, Ttot, ncls] holds the speaker weights of every latent row; every gate of a position in row r adds the blend
w0 E_l[0] + w1 E_l[1] + ... of row r (fp32 products and sums, in that order) where the labelled forward adds
E_l[label]."""
import torch
import torch.nn.functional as F

import oracle_anchored as OA
import oracle_nucleus as ON
import oracle_sampling as OSM
import talkshow_oracle as O


def class_terms(table, style):
    """table [ncls, 2D] (one layer's class_cond_embedding), style [B, H, ncls] -> [B, 2D, H, 1], the class term of every
    position of rows 0..H-1 (the same for both columns), summed in the rule's order."""
    w = style.to(torch.float32)
    acc = w[..., 0:1] * table[0]
    for s in range(1, table.shape[0]):
        acc = acc + w[..., s:s + 1] * table[s]
    return acc.permute(0, 2, 1).unsqueeze(-1)


def pixelcnn_forward(sd, x, style, aud):
    """GatedPixelCNN.forward (gated_pixelcnn_v2.py:130-150, bh_model, eval) with a per-row class term: x [B,H,2] codes,
    style [B,H,ncls], aud [B,256,H,2] -> logits [B,2048,H,2].  The labelled oracle's forward with h[label] replaced by
    class_terms(E_l, style)."""
    e = F.embedding(x.reshape(-1), sd["embedding.weight"]).view(x.shape + (-1,)).permute(0, 3, 1, 2)
    x_v, x_h = e, e
    for l in range(O._n_layers(sd)):
        p = "layers.%d." % l
        k = 7 if l == 0 else 3
        if l == 1:
            a = F.conv2d(aud, sd["embedding_aud.weight"], sd["embedding_aud.bias"])
            x_v = F.conv2d(torch.cat([x_v, a], 1), sd["fusion_v.weight"], sd["fusion_v.bias"])
            x_h = F.conv2d(torch.cat([x_h, a], 1), sd["fusion_h.weight"], sd["fusion_h.bias"])
        wv, wh = sd[p + "vert_stack.weight"], sd[p + "horiz_stack.weight"]
        if l == 0:     # mask A: the vertical stack's own row and the horizontal stack's own column are not seen
            wv = wv.clone()
            wv[:, :, -1].zero_()
            wh = wh.clone()
            wh[:, :, :, -1].zero_()
        h = class_terms(sd[p + "class_cond_embedding.weight"], style)
        h_vert = F.conv2d(x_v, wv, sd[p + "vert_stack.bias"], 1, (k // 2, 1))[:, :, : x_v.size(-2), :]
        out_v = O._gate(h_vert + h)
        h_horiz = F.conv2d(x_h, wh, sd[p + "horiz_stack.bias"], 1, (0, 1))[:, :, :, : x_h.size(-1)]
        v2h = F.conv2d(h_vert, sd[p + "vert_to_horiz.weight"], sd[p + "vert_to_horiz.bias"])
        out = O._gate(v2h + h_horiz + h)
        out_h = F.conv2d(out, sd[p + "horiz_resid.weight"], sd[p + "horiz_resid.bias"])
        if l > 0:
            out_h = out_h + x_h
        x_v, x_h = out_v, out_h
    y = F.relu(F.conv2d(x_h, sd["output_conv.0.weight"], sd["output_conv.0.bias"]))
    return F.conv2d(y, sd["output_conv.2.weight"], sd["output_conv.2.bias"])


def onehot(label, ncls, H):
    """the style schedule [B, H, ncls] of a labelled call"""
    return F.one_hot(label.reshape(-1), ncls).to(torch.float32)[:, None, :].expand(-1, H, -1).contiguous()


def pixelcnn_sample(sd, style, T, B, aud_feat, noise, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, anchors=None,
                    pre_latents=None, pre_audio=None, window=18):
    """The styled sampler: style [B, T0+T, ncls] over every row (the pre_latents prefix first), the draw and anchors of
    oracle_anchored.pixelcnn_sample -> (codes [B,T,2], logp [B,T,2], kept [B,T,2] int32)."""
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
            lg = pixelcnn_forward(sd, x[:, lo:i + 1], style[:, lo:i + 1], aud_feat[:, :, lo:i + 1])[:, :, i - lo, j]
            p = pin[:, i - h0, j]
            code, kn = ON.draw(lg, None if noise is None else noise[step], temperature, top_k, top_p, min_p)
            if anchors is not None:
                code = torch.where(p, anchors[:, i - h0, j], code)
            x[:, i, j] = code
            kept[:, i - h0, j] = torch.where(p, 0, kn)
            logp[:, i - h0, j] = OSM.logp_of(lg, code)
            step += 1
    return x[:, h0:], logp, kept


def body_sample(ckpt, vq_ckpt, mfcc, style, noise, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, anchors=None, window=18):
    """-> (codes, poses [B,4T,C], logp, kept) of the styled body call"""
    B = mfcc.shape[0]
    audio = O.audio_encoder(ckpt["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
    lat, logp, kept = pixelcnn_sample(ckpt["generator"], style, audio.shape[2], B, audio, noise, temperature, top_k, top_p,
                                      min_p, anchors=anchors, window=window)
    body = O.vq_decode(vq_ckpt["g_body"], lat[..., 0])
    hand = O.vq_decode(vq_ckpt["g_hand"], lat[..., 1])
    return lat, torch.cat([body, hand], 1).transpose(1, 2), logp, kept


def score(sd, aud, style, codes):
    """teacher-forced styled forward: aud [B,256,T], style [B,T,ncls], codes [B,T,2] -> (nll [B,T,2], logits
    [B,2048,T,2])"""
    logits = pixelcnn_forward(sd, codes, style, aud.unsqueeze(-1).repeat(1, 1, 1, 2))
    nll = -torch.log_softmax(logits, 1).gather(1, codes.unsqueeze(1))[:, 0]
    return nll, logits
