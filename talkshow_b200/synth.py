"""Checkpoint tensor schema of the TalkSHOW hot path + seeded synthetic checkpoints.

The reference ships no checkpoints in this environment (README.md:73-74 points to external
downloads), so parity is defined on *synthetic* checkpoints written in the reference's own
state-dict format (SURVEY.md Appendix A):

  body-pixel ckpt : {'generator': GatedPixelCNN sd, 'audioencoder': AudioEncoder sd}
                    (nets/smplx_body_pixel.py:104-113)
  body-vq ckpt    : {'g_body': VQVAE(39) sd, 'g_hand': VQVAE(90) sd}   (nets/smplx_body_vq.py:77-94)
  face ckpt       : {'generator': s2g_face.Generator sd}                (nets/base.py:29-36)

Every value is derived from ``torch.rand`` (uniform_) only: that generator is pure
integer->float arithmetic, so the same seed gives bit-identical tensors on any host CPU
(normal_/exponential_ go through vectorised transcendental code that may differ in the last bit
between SIMD code paths).  ``fingerprint`` lets a test prove that.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

# --------------------------------------------------------------------------------------------
# schemas (name -> shape), mirroring the reference modules' state_dict()
# --------------------------------------------------------------------------------------------


def pixelcnn_schema(input_dim=2048, dim=256, n_layers=15, n_classes=4):
    """nets/spg/gated_pixelcnn_v2.py:90-128 (audio=True, bh_model=True)."""
    s = OrderedDict()
    s["embedding_aud.weight"] = (dim, 256, 1, 1)
    s["embedding_aud.bias"] = (dim,)
    for f in ("fusion_v", "fusion_h"):
        s[f + ".weight"] = (dim, 2 * dim, 1, 1)
        s[f + ".bias"] = (dim,)
    s["embedding.weight"] = (input_dim, dim)
    for l in range(n_layers):
        k = 7 if l == 0 else 3
        p = "layers.%d." % l
        s[p + "class_cond_embedding.weight"] = (n_classes, 2 * dim)
        s[p + "vert_stack.weight"] = (2 * dim, dim, k // 2 + 1, 3)
        s[p + "vert_stack.bias"] = (2 * dim,)
        s[p + "vert_to_horiz.weight"] = (2 * dim, 2 * dim, 1, 1)
        s[p + "vert_to_horiz.bias"] = (2 * dim,)
        s[p + "horiz_stack.weight"] = (2 * dim, dim, 1, 2)
        s[p + "horiz_stack.bias"] = (2 * dim,)
        s[p + "horiz_resid.weight"] = (dim, dim, 1, 1)
        s[p + "horiz_resid.bias"] = (dim,)
    s["output_conv.0.weight"] = (512, dim, 1, 1)
    s["output_conv.0.bias"] = (512,)
    s["output_conv.2.weight"] = (input_dim, 512, 1, 1)
    s["output_conv.2.bias"] = (input_dim,)
    return s


def _cnr(s, p, cin, cout, k, residual=None, transpose=False):
    """vqvae_modules.ConvNormRelu (nets/spg/vqvae_modules.py:87-172): conv + BatchNorm1d
    (+ residual conv).  ConvTranspose1d weights are [C_in, C_out, k]."""
    if residual:
        s[p + "residual_layer.weight"] = (cin, cout, k) if transpose else (cout, cin, k)
        s[p + "residual_layer.bias"] = (cout,)
    s[p + "conv.weight"] = (cin, cout, k) if transpose else (cout, cin, k)
    s[p + "conv.bias"] = (cout,)
    _bn(s, p + "norm.", cout)


def _bn(s, p, c):
    s[p + "weight"] = (c,)
    s[p + "bias"] = (c,)
    s[p + "running_mean"] = (c,)
    s[p + "running_var"] = (c,)
    s[p + "num_batches_tracked"] = ()


def _stack(s, p, c, layers=2):
    """Res_CNR_Stack (nets/spg/vqvae_modules.py:175-212)."""
    for i in range(layers):
        _cnr(s, p + "_layers.%d." % i, c, c, 3)
    s[p + "conv.weight"] = (c, c, 3)
    s[p + "conv.bias"] = (c,)
    _bn(s, p + "norm.", c)


def _encoder(s, p, in_dim, hid):
    _cnr(s, p + "project.", in_dim, hid // 4, 3)
    _stack(s, p + "_enc_1.", hid // 4)
    _cnr(s, p + "_down_1.", hid // 4, hid // 2, 4, residual=True)
    _stack(s, p + "_enc_2.", hid // 2)
    _cnr(s, p + "_down_2.", hid // 2, hid, 4, residual=True)
    _stack(s, p + "_enc_3.", hid)


def audioenc_schema(in_dim=64, hid=256):
    """AudioEncoder (nets/spg/vqvae_1d.py:11-34)."""
    s = OrderedDict()
    _encoder(s, "", in_dim, hid)
    return s


def vqvae_schema(in_dim, emb=64, codes=2048, hid=1024):
    """VQVAE (nets/spg/vqvae_1d.py:168-208): Encoder :66-92, VectorQuantizerEMA, Decoder :116-149."""
    s = OrderedDict()
    _encoder(s, "encoder.", in_dim, hid)
    s["encoder.pre_vq_conv.weight"] = (emb, hid, 1)
    s["encoder.pre_vq_conv.bias"] = (emb,)
    s["vq_layer.embeddings"] = (codes, emb)
    s["vq_layer.ema_dw.hidden"] = (codes, emb)
    s["vq_layer.ema_cluster_size.hidden"] = (codes,)
    s["decoder.aft_vq_conv.weight"] = (hid, emb, 1)
    s["decoder.aft_vq_conv.bias"] = (hid,)
    _stack(s, "decoder._dec_1.", hid)
    _cnr(s, "decoder._up_2.", hid, hid // 2, 4, residual=True, transpose=True)
    _stack(s, "decoder._dec_2.", hid // 2)
    _cnr(s, "decoder._up_3.", hid // 2, hid // 4, 4, residual=True, transpose=True)
    _stack(s, "decoder._dec_3.", hid // 4)
    s["decoder.project.weight"] = (in_dim, hid // 4, 1)
    s["decoder.project.bias"] = (in_dim,)
    return s


W2V_CONV_KERNEL = (10, 3, 3, 3, 3, 2, 2)
W2V_CONV_STRIDE = (5, 2, 2, 2, 2, 2, 2)


def face_schema(n_classes=4, jaw_dim=3, exp_dim=100, identity=True):
    """s2g_face.Generator (nets/spg/s2g_face.py:142-194) with the HF wav2vec2-base encoder
    (transformers Wav2Vec2Model; names of the installed 5.x version, where the positional conv
    carries a weight_norm parametrisation ``parametrizations.weight.original{0,1}`` = (g, v)).
    ``identity=False`` is the convert_to_6d net (nets/smplx_face.py:37-45): AudioEncoder(256, 256, identity=False)
    has no id_mlp, and first_net layer 0 maps 256 -> 256 with an nn.Identity residual (nets/layers.py:95-96)."""
    s = OrderedDict()
    a = "audio_encoder."
    s[a + "masked_spec_embed"] = (768,)
    for i, k in enumerate(W2V_CONV_KERNEL):
        s[a + "feature_extractor.conv_layers.%d.conv.weight" % i] = (512, 1 if i == 0 else 512, k)
        if i == 0:
            s[a + "feature_extractor.conv_layers.0.layer_norm.weight"] = (512,)
            s[a + "feature_extractor.conv_layers.0.layer_norm.bias"] = (512,)
    s[a + "feature_projection.layer_norm.weight"] = (512,)
    s[a + "feature_projection.layer_norm.bias"] = (512,)
    s[a + "feature_projection.projection.weight"] = (768, 512)
    s[a + "feature_projection.projection.bias"] = (768,)
    e = a + "encoder."
    s[e + "pos_conv_embed.conv.bias"] = (768,)
    s[e + "pos_conv_embed.conv.parametrizations.weight.original0"] = (1, 1, 128)
    s[e + "pos_conv_embed.conv.parametrizations.weight.original1"] = (768, 48, 128)
    s[e + "layer_norm.weight"] = (768,)
    s[e + "layer_norm.bias"] = (768,)
    for l in range(12):
        p = e + "layers.%d." % l
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            s[p + "attention.%s.weight" % n] = (768, 768)
            s[p + "attention.%s.bias" % n] = (768,)
        s[p + "layer_norm.weight"] = (768,)
        s[p + "layer_norm.bias"] = (768,)
        s[p + "feed_forward.intermediate_dense.weight"] = (3072, 768)
        s[p + "feed_forward.intermediate_dense.bias"] = (3072,)
        s[p + "feed_forward.output_dense.weight"] = (768, 3072)
        s[p + "feed_forward.output_dense.bias"] = (768,)
        s[p + "final_layer_norm.weight"] = (768,)
        s[p + "final_layer_norm.bias"] = (768,)
    s["audio_feature_map.weight"] = (256, 768)
    s["audio_feature_map.bias"] = (256,)
    f = "audio_middle.first_net.conv_layers."
    if identity:
        s["audio_middle.id_mlp.weight"] = (64, n_classes, 1)
        s["audio_middle.id_mlp.bias"] = (64,)
        s[f + "0.residual_layer.0.weight"] = (256, 320, 3)
        s[f + "0.residual_layer.0.bias"] = (256,)
    for i, cin in enumerate((320 if identity else 256, 256, 256)):
        s[f + "%d.conv.weight" % i] = (256, cin, 3)
        s[f + "%d.conv.bias" % i] = (256,)
        s[f + "%d.norm.weight" % i] = (256,)
        s[f + "%d.norm.bias" % i] = (256,)
    for n, shp in (("weight_ih_l0", (768, 256)), ("weight_hh_l0", (768, 256)), ("bias_ih_l0", (768,)),
                   ("bias_hh_l0", (768,))):
        s["audio_middle.grus." + n] = shp  # present in the dict, unused in forward (s2g_face.py:134-137)
    for b, c in ((0, 64), (1, 256)):
        for i in range(3):
            cin = 256 if i == 0 else c
            p = "decoder.%d.%d." % (b, i)
            s[p + "conv.weight"] = (c, cin, 3)
            s[p + "conv.bias"] = (c,)
            s[p + "norm.weight"] = (c,)
            s[p + "norm.bias"] = (c,)
    s["final_out.0.weight"] = (jaw_dim, 64, 1)
    s["final_out.0.bias"] = (jaw_dim,)
    s["final_out.1.weight"] = (exp_dim, 256, 1)
    s["final_out.1.bias"] = (exp_dim,)
    return s


# --------------------------------------------------------------------------------------------
# seeded fill
# --------------------------------------------------------------------------------------------


def _u(gen, shape, lo, hi):
    return torch.rand(shape, generator=gen, dtype=torch.float32) * (hi - lo) + lo


def _fill(name, shape, gen, transpose_conv=False):
    """Deterministic value rule by tensor role (suffix of the name)."""
    if name.endswith("num_batches_tracked"):
        return torch.zeros((), dtype=torch.int64)
    if name.endswith("running_var"):
        return _u(gen, shape, 0.5, 1.5)
    if name.endswith("running_mean"):
        return _u(gen, shape, -0.17, 0.17)
    if name.endswith("masked_spec_embed"):
        return _u(gen, shape, 0.0, 1.0)
    if name.endswith("original0"):                       # weight_norm g
        return _u(gen, shape, 0.8, 1.6)
    if "norm" in name.split(".")[-2] and name.endswith(".weight") and len(shape) == 1:
        return _u(gen, shape, 0.8, 1.2)                   # BN / LN / GN gamma
    if "norm" in name.split(".")[-2] and name.endswith(".bias"):
        return _u(gen, shape, -0.17, 0.17)
    if name.endswith("vq_layer.embeddings"):
        # the reference initialises xavier_uniform_ (vqvae_modules.py:266-268) and EMA training then
        # moves the codes onto the encoder's output range; +-0.5 matches the synthetic encoders'
        # output spread so that argmin picks varied codes (xavier scale would pick one code always)
        return _u(gen, shape, -0.5, 0.5)
    if "ema_" in name:
        return torch.zeros(shape, dtype=torch.float32)
    if name.endswith("embedding.weight") and len(shape) == 2:
        return _u(gen, shape, -1.73, 1.73)                # unit variance like nn.Embedding's N(0,1)
    if name.endswith(".bias") or name.startswith("audio_middle.grus.bias"):
        return _u(gen, shape, -0.05, 0.05)
    # conv / linear weight: xavier-uniform bound on (fan_in, fan_out)
    rf = 1
    for d in shape[2:]:
        rf *= d
    if len(shape) == 1:
        return _u(gen, shape, -0.05, 0.05)
    fan_out, fan_in = shape[0] * rf, shape[1] * rf
    a = math.sqrt(6.0 / (fan_in + fan_out))
    return _u(gen, shape, -a, a)


def synth_state(schema, seed, scale=None):
    gen = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, shape in schema.items():
        t = _fill(name, tuple(shape), gen)
        if scale and name in scale:
            t = t * scale[name]
        sd[name] = t
    return sd


def pixelcnn_state(seed=0, logit_scale=8.0, **kw):
    """``logit_scale`` sharpens the output layer so sampled distributions look like a trained
    prior rather than near-uniform (SURVEY.md §7 hard part 1)."""
    sd = synth_state(pixelcnn_schema(**kw), seed, scale={"output_conv.2.weight": logit_scale})
    # mask 'A' taps are zeroed in place by the reference at every forward
    # (gated_pixelcnn_v2.py:57-59); a trained checkpoint therefore stores zeros there.
    sd["layers.0.vert_stack.weight"][:, :, -1].zero_()
    sd["layers.0.horiz_stack.weight"][:, :, :, -1].zero_()
    return sd


def audioenc_state(seed=1):
    return synth_state(audioenc_schema(), seed)


def vqvae_state(in_dim, seed):
    return synth_state(vqvae_schema(in_dim), seed)


def face_state(seed=4):
    return synth_state(face_schema(), seed)


def body_pixel_checkpoint(seed=0):
    """What ``torch.load(ckpt)['generator']`` holds for s2g_body_pixel (smplx_body_pixel.py:104-113)."""
    return {"generator": pixelcnn_state(seed), "audioencoder": audioenc_state(seed + 1)}


def body_pixel_checkpoint_6d(seed=0):
    """convert_to_6d geometry of nets/smplx_body_pixel.py:49-52: pixelcnn(2048, 512, 10, 4, True, True)."""
    return {"generator": pixelcnn_state(seed + 20, dim=512, n_layers=10), "audioencoder": audioenc_state(seed + 1)}


def body_vq_checkpoint_6d(seed=0):
    """VQ-VAEs over the 6-D pose layout: body 78, hands 180 channels (nets/smplx_body_pixel.py:54-57 with scale 2)."""
    return {"g_body": vqvae_state(78, seed + 22), "g_hand": vqvae_state(180, seed + 23)}


def body_vq_checkpoint(seed=0):
    """... for s2g_body_vq, also the file ``config.Model.vq_path`` points to."""
    return {"g_body": vqvae_state(39, seed + 2), "g_hand": vqvae_state(90, seed + 3)}


def face_checkpoint(seed=0):
    return {"generator": face_state(seed + 4)}


def face_checkpoint_6d(seed=0):
    """convert_to_6d face (nets/smplx_face.py:37-45, init_params scale 2): identity-free net, 6-D jaw head."""
    return {"generator": synth_state(face_schema(identity=False, jaw_dim=6), seed + 24)}


def fingerprint(sd):
    """Order-independent checksum of a (possibly nested) state dict: float64 sum and abs-sum."""
    tot = 0.0
    ab = 0.0
    n = 0
    stack = [sd]
    while stack:
        d = stack.pop()
        for v in d.values():
            if isinstance(v, dict):
                stack.append(v)
            elif torch.is_tensor(v) and v.is_floating_point():
                tot += float(v.double().sum())
                ab += float(v.double().abs().sum())
                n += v.numel()
    return {"n": n, "sum": tot, "abs": ab}


# --------------------------------------------------------------------------------------------
# synthetic inputs (SURVEY.md §8d)
# --------------------------------------------------------------------------------------------


def synth_wave(B, N, seed=1234):
    """16 kHz mono: 0.1*uniform-noise (unit-variance scaled) + 220 Hz sine, computed in float64
    then rounded, so it is identical on every host."""
    gen = torch.Generator().manual_seed(seed)
    noise = (torch.rand((B, N), generator=gen, dtype=torch.float64) - 0.5) * math.sqrt(12.0) * 0.1
    t = torch.arange(N, dtype=torch.float64) / 16000.0
    phase = torch.arange(B, dtype=torch.float64)[:, None] * 0.37
    return (noise + 0.2 * torch.sin(2 * math.pi * 220.0 * t[None, :] + phase)).float()


def synth_mfcc(B, M, seed=1234):
    """Stand-in MFCC features [B, 64, M] with roughly the dynamic range torchaudio's MFCC has on
    speech, divided by ~10 (c0 negative, decaying spread).  Pure uniform arithmetic (host independent)."""
    gen = torch.Generator().manual_seed(seed + 7)
    x = (torch.rand((B, 64, M), generator=gen, dtype=torch.float32) - 0.5) * 2.0
    scale = 4.0 / (1.0 + 0.25 * torch.arange(64, dtype=torch.float32))[None, :, None]
    x = x * scale
    x[:, 0, :] -= 6.0
    return x


def synth_poses(B, F, seed=1234):
    """Axis-angle scale SMPL-X pose block [B, 165, F] (config 2): per-channel sum of three slow
    sinusoids (periods 16-80 frames) plus small jitter, so that the 4x-downsampled latent sequence
    moves through the codebook instead of sitting on one code.  float64 math, rounded once."""
    gen = torch.Generator().manual_seed(seed + 11)
    t = torch.arange(F, dtype=torch.float64)[None, None, None, :]
    amp = torch.rand((B, 165, 3, 1), generator=gen, dtype=torch.float64) * 0.6
    per = 16.0 + torch.rand((B, 165, 3, 1), generator=gen, dtype=torch.float64) * 64.0
    ph = torch.rand((B, 165, 3, 1), generator=gen, dtype=torch.float64) * 2 * math.pi
    x = (amp * torch.sin(2 * math.pi * t / per + ph)).sum(2)
    x = x + (torch.rand((B, 165, F), generator=gen, dtype=torch.float64) - 0.5) * 0.1
    return x.float()
