"""Thin object wrapper over the C ABI: PyTorch CUDA tensors in, PyTorch CUDA tensors out.

Module-level mirror of the reference network modules (nets/spg/*.py) — used by the wrapper classes
in talkshow_b200/nets/ and directly by the parity tests.  Every method enqueues on the current
CUDA stream of the engine's device and returns without synchronising.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib

PIX_TILE = 64  # samples per PixelCNN launch (csrc/pixelcnn.h PIX_MB)
NCODE = 2048   # codes of the body prior


def check_sample_controls(temperature, top_k, top_p=1.0, min_p=0.0):
    """Validate the values of the sampler's controls (ValueError): temperature finite and >= 0 (0 = greedy decoding),
    top_k an integer in [0, 2048] (0 = off), top_p in (0, 1] (1 = off), min_p in [0, 1] (0 = off)."""
    try:
        t = float(temperature)
    except (TypeError, ValueError):
        raise ValueError("temperature must be a number, got %r" % (temperature,))
    if not math.isfinite(t) or t < 0:
        raise ValueError("temperature must be finite and >= 0 (0 = greedy), got %r" % (temperature,))
    if isinstance(top_k, bool) or int(top_k) != top_k or not 0 <= int(top_k) <= NCODE:
        raise ValueError("top_k must be an integer in [0, %d] (0 = off), got %r" % (NCODE, top_k))
    for name, v, ok in (("top_p", top_p, lambda x: 0 < x <= 1), ("min_p", min_p, lambda x: 0 <= x <= 1)):
        try:
            x = float(v)
        except (TypeError, ValueError):
            raise ValueError("%s must be a number, got %r" % (name, v))
        # the engine takes the fp32 value: one that rounds out of the range (a top_p below the smallest float) is invalid too
        if isinstance(v, bool) or not ok(x) or not ok(float(torch.tensor(x, dtype=torch.float32))):
            raise ValueError("%s must lie in %s, got %r" % (name, "(0, 1] (1 = off)" if name == "top_p" else "[0, 1] (0 = off)", v))


def sample_controls(temperature=1.0, top_k=0, keep_logp=False, top_p=1.0, min_p=0.0):
    """Validated keyword arguments of ``Engine.pixelcnn_generate`` / ``body_generate`` for these controls; empty at the
    defaults, so that those calls keep the default entry points (ts_pixelcnn_generate / ts_body_generate).  ``top_p``,
    ``min_p`` and ``want_kept`` appear only when nucleus or min-p truncation is on; the keep-set sizes are then asked for
    together with the log-likelihoods.  Per-clip controls (``check_clip_controls``) give all four as float32 / int32
    arrays [B], with ``want_kept`` when any clip truncates by top_p or min_p."""
    if per_clip(temperature, top_k, top_p, min_p):
        cc = check_clip_controls(temperature, top_k, top_p, min_p)
        nucleus = bool((cc["top_p"] < 1.0).any() or (cc["min_p"] > 0.0).any())
        return dict(temperature=cc["temperature"], top_k=cc["top_k"], want_logp=bool(keep_logp), top_p=cc["top_p"],
                    min_p=cc["min_p"], want_kept=bool(keep_logp) and nucleus)
    check_sample_controls(temperature, top_k, top_p, min_p)
    nucleus = float(top_p) < 1.0 or float(min_p) > 0.0
    if float(temperature) == 1.0 and not top_k and not keep_logp and not nucleus:
        return {}
    ctl = dict(temperature=temperature, top_k=top_k, want_logp=bool(keep_logp))
    if nucleus:
        ctl.update(top_p=top_p, min_p=min_p, want_kept=bool(keep_logp))
    return ctl


# one entry of the per-clip controls (include/talkshow_b200.h ts_clip_ctl)
CLIP_CTL = np.dtype([("temperature", "<f4"), ("top_k", "<i4"), ("top_p", "<f4"), ("min_p", "<f4")])


def _is_per_clip(v):
    """A control given per clip: a list / tuple, or a numpy array or tensor with a dimension (a 0-d one is a scalar)."""
    if torch.is_tensor(v) or isinstance(v, np.ndarray):
        return v.ndim > 0
    return isinstance(v, (list, tuple))


def per_clip(temperature, top_k, top_p=1.0, min_p=0.0):
    """True when any of the four sampling controls is given per clip (``check_clip_controls``)."""
    return any(_is_per_clip(v) for v in (temperature, top_k, top_p, min_p))


def check_clip_controls(temperature, top_k, top_p=1.0, min_p=0.0, B=None):
    """Per-clip sampling controls as a host array [B] of ``CLIP_CTL`` (ts_clip_ctl).  Each control is a scalar, broadcast
    to every clip, or a length-B sequence / 1-D numpy array / 1-D tensor; B defaults to the length of the per-clip
    values.  Every clip's values follow ``check_sample_controls`` (fp32 rounding of top_p / min_p included) and a
    temperature must stay finite in fp32.  A bool element, another shape or another length raises ValueError; an
    element's error names its clip."""
    cols = {}
    for name, v in (("temperature", temperature), ("top_k", top_k), ("top_p", top_p), ("min_p", min_p)):
        if not _is_per_clip(v):
            continue
        if torch.is_tensor(v) or isinstance(v, np.ndarray):
            if v.ndim != 1:
                raise ValueError("%s: per-clip values must be one-dimensional, got shape %s" % (name, tuple(v.shape)))
            v = v.tolist()
        v = list(v)
        if B is None:
            B = len(v)
        if len(v) != B:
            raise ValueError("%s: %d per-clip values for %d clips" % (name, len(v), B))
        for b, x in enumerate(v):
            if isinstance(x, bool):
                raise ValueError("%s: clip %d: a bool is not a sampling control, got %r" % (name, b, x))
        cols[name] = v
    if B is None:
        raise ValueError("check_clip_controls: no per-clip value and no batch size")
    scalars = dict(temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p)
    defaults = dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0)
    check_sample_controls(**{n: defaults[n] if n in cols else v for n, v in scalars.items()})   # the broadcast scalars
    out = np.zeros(B, CLIP_CTL)
    for b in range(B):
        t, k, p, m = (cols[n][b] if n in cols else scalars[n] for n in ("temperature", "top_k", "top_p", "min_p"))
        try:
            check_sample_controls(t, k, p, m)
            with np.errstate(over="ignore"):
                t32 = np.float32(float(t))
            if not math.isfinite(t32):
                raise ValueError("temperature must be finite in fp32, got %r" % (t,))
        except ValueError as ex:
            raise ValueError("clip %d: %s" % (b, ex)) from None
        out[b] = (float(t), int(k), float(p), float(m))
    return out


# one entry of the per-clip logit shaping (include/talkshow_b200.h ts_clip_shape)
CLIP_SHAPE = np.dtype([("repetition_penalty", "<f4"), ("repetition_window", "<i4")])
BIAS_MAX = 1e4   # largest |value| of a finite code bias


def _clip_values(name, v, B):
    """A per-clip value as a list of B elements (a length-B sequence, 1-D numpy array or 1-D tensor); a bool element, another
    shape or another length raises ValueError."""
    if torch.is_tensor(v) or isinstance(v, np.ndarray):
        if v.ndim != 1:
            raise ValueError("%s: per-clip values must be one-dimensional, got shape %s" % (name, tuple(v.shape)))
        v = v.tolist()
    v = list(v)
    if len(v) != B:
        raise ValueError("%s: %d per-clip values for %d clips" % (name, len(v), B))
    for b, x in enumerate(v):
        if isinstance(x, bool):
            raise ValueError("%s: clip %d: a bool is not a shaping value, got %r" % (name, b, x))
    return v


def _check_shape_values(penalty, window):
    """ValueError unless the repetition penalty is a number, finite and >= 1 in fp32, and the window an integer in
    [1, 2^31 - 1]."""
    try:
        if isinstance(penalty, bool):
            raise TypeError
        with np.errstate(over="ignore"):
            p32 = np.float32(float(penalty))
    except (TypeError, ValueError):
        raise ValueError("repetition_penalty must be a number, got %r" % (penalty,)) from None
    if not (math.isfinite(p32) and p32 >= 1.0):
        raise ValueError("repetition_penalty must be finite and >= 1 (1 = off), got %r" % (penalty,))
    try:
        if isinstance(window, bool) or int(window) != window:
            raise TypeError
    except (TypeError, ValueError):
        raise ValueError("repetition_window must be an integer, got %r" % (window,)) from None
    if not 1 <= int(window) <= 2 ** 31 - 1:
        raise ValueError("repetition_window must lie in [1, 2^31 - 1] latent rows, got %r" % (window,))


def check_clip_shape(repetition_penalty=1.0, repetition_window=8, B=None):
    """Per-clip logit shaping as a host array [B] of ``CLIP_SHAPE`` (ts_clip_shape).  Each value is a scalar, broadcast to
    every clip, or a length-B sequence / 1-D numpy array / 1-D tensor (B defaults to its length).  The penalty must be
    finite and >= 1 in fp32 (1 = off), the window an integer >= 1 (latent rows).  A bool element, another shape or another
    length raises ValueError; an element's error names its clip."""
    cols = {}
    for name, v in (("repetition_penalty", repetition_penalty), ("repetition_window", repetition_window)):
        if _is_per_clip(v):
            if B is None:
                B = len(v)
            cols[name] = _clip_values(name, v, B)
    if B is None:
        raise ValueError("check_clip_shape: no per-clip value and no batch size")
    scalars = dict(repetition_penalty=repetition_penalty, repetition_window=repetition_window)
    defaults = dict(repetition_penalty=1.0, repetition_window=8)
    _check_shape_values(*(defaults[n] if n in cols else v for n, v in scalars.items()))   # the broadcast scalars
    out = np.zeros(B, CLIP_SHAPE)
    for b in range(B):
        p, w = (cols[n][b] if n in cols else scalars[n] for n in ("repetition_penalty", "repetition_window"))
        try:
            _check_shape_values(p, w)
        except ValueError as ex:
            raise ValueError("clip %d: %s" % (b, ex)) from None
        out[b] = (float(p), int(w))
    return out


def check_code_bias(code_bias, B):
    """Code bias of a shaped call as a float32 tensor [B,2,2048] (host or device, as given): a float or integer tensor or
    numpy array of shape [B,2,2048], or [2,2048] (the same two rows for every clip).  Column 0 biases the body codebook,
    column 1 the hand codebook.  After conversion to float32 every value must be finite with |v| <= 1e4, or -inf (the code
    is never drawn), and every (clip, column) row must keep a finite value.  Anything else raises ValueError naming the
    clip and column.  The value check of a device tensor reads one reduction back: one synchronisation."""
    if isinstance(code_bias, np.ndarray):
        if code_bias.dtype.kind not in "fiu":
            raise ValueError("code_bias must be a float array [%d,2,%d] or [2,%d], got dtype %s" % (B, NCODE, NCODE, code_bias.dtype))
        code_bias = torch.from_numpy(np.ascontiguousarray(code_bias))
    if not torch.is_tensor(code_bias):
        raise ValueError("code_bias must be a float tensor or numpy array [%d,2,%d] or [2,%d], got %r"
                         % (B, NCODE, NCODE, type(code_bias)))
    if code_bias.dtype == torch.bool or code_bias.is_complex():
        raise ValueError("code_bias must be a float tensor, got %s" % (code_bias.dtype,))
    code_bias = code_bias.to(torch.float32)
    if tuple(code_bias.shape) == (2, NCODE):
        code_bias = code_bias.expand(B, 2, NCODE)
    if tuple(code_bias.shape) != (B, 2, NCODE):
        raise ValueError("code_bias must have shape [%d,2,%d] or [2,%d], got %s" % (B, NCODE, NCODE, tuple(code_bias.shape)))
    code_bias = code_bias.contiguous()
    fin = torch.isfinite(code_bias)
    bad = torch.isnan(code_bias) | (code_bias == float("inf")) | (fin & (code_bias.abs() > BIAS_MAX))
    flags = torch.stack([bad.any(-1), ~fin.any(-1)], -1).cpu()          # [B,2,2]: one read back
    if flags.any():
        b, c, k = (int(i) for i in torch.nonzero(flags)[0])
        what = ("values must be finite with |v| <= %g, or -inf" % BIAS_MAX if k == 0
                else "every code is -inf: the draw keeps no code")
        raise ValueError("code_bias: clip %d, column %d (%s): %s" % (b, c, ("body", "hand")[c], what))
    return code_bias


def shaping_kwargs(repetition_penalty=1.0, repetition_window=8, code_bias=None, B=None):
    """The shaping keywords a caller forwards to ``Engine.pixelcnn_generate`` / ``body_generate``: none when the call
    shapes nothing (no code_bias, repetition_penalty 1 for every clip), so that such calls forward what they forwarded
    before.  The penalty and window are validated here (``check_clip_shape``), the bias by the engine."""
    shape = check_clip_shape(repetition_penalty, repetition_window, B)
    if code_bias is None and not (shape["repetition_penalty"] != 1.0).any():
        return {}
    return dict(repetition_penalty=repetition_penalty, repetition_window=repetition_window, code_bias=code_bias)


GUIDANCE_MAX = 100.0   # largest guidance scale (include/talkshow_b200.h TS_GUIDANCE_MAX)
GUIDE_PAIRS = PIX_TILE // 2   # pairs per guided launch: two branches each, one 64-sample tile


def check_guidance(guidance, B):
    """Guidance scales of a guided call as a float32 host array [B]: a scalar, applied to every clip, or one value per clip
    (a length-B sequence, 1-D numpy array or 1-D tensor).  Each value must be a number whose fp32 value is finite and in
    [0, 100] (1 = no guidance).  Anything else raises ValueError naming the clip."""
    vals = _clip_values("guidance", guidance, B) if _is_per_clip(guidance) else [guidance] * B
    out = np.zeros(B, np.float32)
    for b, w in enumerate(vals):
        try:
            if isinstance(w, bool):
                raise TypeError
            with np.errstate(over="ignore"):
                w32 = np.float32(float(w))
        except (TypeError, ValueError):
            raise ValueError("guidance: clip %d: must be a number, got %r" % (b, w)) from None
        if not (math.isfinite(w32) and 0.0 <= w32 <= GUIDANCE_MAX):
            raise ValueError("guidance: clip %d: must be finite and in [0, %g] (1 = no guidance), got %r" % (b, GUIDANCE_MAX, w))
        out[b] = w32
    return out


def guide_kwargs(guidance=None, guide_mfcc=None, guide_label=None, guide_style=None, keep_logp=False, engine=None, B=None,
                 M=None):
    """The guidance keywords a caller forwards to ``Engine.body_generate``: none without ``guidance`` (the call then
    forwards what it forwarded before; a negative conditioning without guidance raises ValueError).  ``guide_mfcc`` may be
    the string "silence": ``engine.silence_mfcc(M, B)``.  ``keep_logp`` asks for the negative branches' log p too."""
    if guidance is None:
        if guide_mfcc is not None or guide_label is not None or guide_style is not None:
            raise ValueError("a negative conditioning (guide_mfcc / guide_id / guide_style) needs guidance")
        return {}
    if isinstance(guide_mfcc, str):
        if guide_mfcc != "silence":
            raise ValueError("guide_mfcc: the only named conditioning is \"silence\", got %r" % (guide_mfcc,))
        guide_mfcc = engine.silence_mfcc(M, B)
    return dict(guidance=guidance, guide_mfcc=guide_mfcc, guide_label=guide_label, guide_style=guide_style,
                want_guide_logp=bool(keep_logp))


def _same_input(a, b):
    """Whether a negative-conditioning field repeats the clip's own, decided without a device synchronisation: the same
    object, equal host values (a one-element label broadcast), or a device tensor viewing the same memory.  Two device
    tensors with equal values in different memory count as different."""
    if a is b:
        return True
    if torch.is_tensor(a) and a.is_cuda or torch.is_tensor(b) and b.is_cuda:
        return (torch.is_tensor(a) and torch.is_tensor(b) and a.device == b.device and a.dtype == b.dtype
                and a.shape == b.shape and a.stride() == b.stride() and a.data_ptr() == b.data_ptr())
    a, b = torch.as_tensor(np.asarray(a)), torch.as_tensor(np.asarray(b))
    try:
        a, b = torch.broadcast_tensors(a, b)
    except RuntimeError:
        return False
    return bool(torch.equal(a, b.to(a.dtype)))


def _interleave(x, g):
    """Rows b of x and g as rows 2b and 2b + 1 of one tensor (the branches of a guided call)."""
    return torch.stack([x, g], 1).reshape((2 * x.shape[0],) + tuple(x.shape[1:])).contiguous()


def sampled(temperature):
    """True when a call with this (validated) temperature draws noise: temperature > 0, for some clip when per clip."""
    if _is_per_clip(temperature):
        vals = temperature.tolist() if hasattr(temperature, "tolist") else temperature
        return any(float(t) > 0 for t in vals)
    return float(temperature) > 0


def _wrap64(v):
    """An integer as the int64 with the same low 64 bits."""
    return (int(v) + (1 << 63)) % (1 << 64) - (1 << 63)


def clip_seeds(seed, B):
    """Per-clip seeds of a batch from one integer: ``seed + arange(B)`` wrapped to int64 bits, int64 [B] (host)."""
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise ValueError("clip_seeds: seed must be an integer, got %r" % (seed,))
    return torch.tensor([_wrap64(int(seed) + b) for b in range(int(B))], dtype=torch.int64)


def check_seeds(seeds, B):
    """Seeds of a seeded call as an int64 tensor [B]: an int64 tensor of shape [B] (host or device) is taken as it is, a
    length-B sequence of integers is wrapped to int64 bits.  Any other shape, dtype or type raises ValueError."""
    if torch.is_tensor(seeds):
        if seeds.dtype != torch.int64 or tuple(seeds.shape) != (B,):
            raise ValueError("seeds must be an int64 tensor of shape [%d], got %s %s" % (B, seeds.dtype, tuple(seeds.shape)))
        return seeds
    if isinstance(seeds, np.ndarray):
        if seeds.dtype.kind not in "iu" or seeds.shape != (B,):
            raise ValueError("seeds must be an integer array of shape [%d], got %s %s" % (B, seeds.dtype, seeds.shape))
        seeds = seeds.tolist()
    if isinstance(seeds, (str, bytes)) or not hasattr(seeds, "__len__") or len(seeds) != B:
        raise ValueError("seeds must be a sequence of %d integers or an int64 tensor [%d], got %r" % (B, B, seeds))
    if any(isinstance(s, bool) or not isinstance(s, (int, np.integer)) for s in seeds):
        raise ValueError("seeds must be integers, got %r" % (seeds,))
    return torch.tensor([_wrap64(s) for s in seeds], dtype=torch.int64)


def resolve_clip_seeds(value, B):
    """The ``clip_seeds=`` keyword of the wrappers: None stays None, an integer means ``clip_seeds(value, B)``, a length-B
    sequence or tensor gives one seed per clip (``check_seeds``)."""
    if value is None:
        return None
    if isinstance(value, (int, np.integer)) and not isinstance(value, bool):
        return clip_seeds(value, B)
    return check_seeds(value, B)


def check_anchors(anchors, B, T):
    """Anchors of an anchored call as an int64 tensor [B,T,2] (host or device, as given): an int64 tensor or a numpy
    integer array of that shape whose values lie in [-1, 2048) (-1 = sample the draw, a code = pin it).  Anything else
    raises ValueError.  The value check of a device tensor reads one reduction back: one synchronisation."""
    if isinstance(anchors, np.ndarray):
        if anchors.dtype.kind not in "iu" or anchors.shape != (B, T, 2):
            raise ValueError("anchors must be an integer array of shape [%d,%d,2], got %s %s" % (B, T, anchors.dtype, anchors.shape))
        if anchors.size and (anchors.min() < -1 or anchors.max() >= NCODE):
            raise ValueError("anchors must lie in [-1, %d) (-1 = sampled), got values in [%d, %d]"
                             % (NCODE, anchors.min(), anchors.max()))
        return torch.from_numpy(np.ascontiguousarray(anchors, dtype=np.int64))
    if not torch.is_tensor(anchors):
        raise ValueError("anchors must be an int64 tensor or an integer numpy array [%d,%d,2], got %r" % (B, T, type(anchors)))
    if anchors.dtype != torch.int64 or tuple(anchors.shape) != (B, T, 2):
        raise ValueError("anchors must be an int64 tensor of shape [%d,%d,2], got %s %s" % (B, T, anchors.dtype, tuple(anchors.shape)))
    if anchors.numel():
        lo, hi = (int(v) for v in torch.stack([anchors.min(), anchors.max()]).tolist())
        if lo < -1 or hi >= NCODE:
            raise ValueError("anchors must lie in [-1, %d) (-1 = sampled), got values in [%d, %d]" % (NCODE, lo, hi))
    return anchors


def check_style(style, B, Ttot, ncls):
    """Speaker schedule of a styled call as a float32 tensor [B,Ttot,ncls] (host or device, as given): a float tensor or
    numpy array of shape [B,Ttot,ncls], or [B,ncls] (one mixture per clip, broadcast over the rows).  It is converted to
    float32 first and the float32 values are checked: finite, >= 0, each row summing to 1 within 1e-5 (a convex mixture of
    the prior's trained speaker embeddings).  Anything else raises ValueError.  A device tensor costs one
    synchronisation."""
    if isinstance(style, np.ndarray):
        if style.dtype.kind != "f":
            raise ValueError("style must be a floating-point array, got %s" % (style.dtype,))
        style = torch.from_numpy(np.ascontiguousarray(style))
    if not torch.is_tensor(style):
        raise ValueError("style must be a float tensor or numpy array [%d,%d,%d] or [%d,%d], got %r"
                         % (B, Ttot, ncls, B, ncls, type(style)))
    if not style.is_floating_point():
        raise ValueError("style must be a floating-point tensor, got %s" % (style.dtype,))
    shape = tuple(style.shape)
    if shape == (B, ncls):
        style = style[:, None, :].expand(B, Ttot, ncls)
    elif shape != (B, Ttot, ncls):
        raise ValueError("style must have shape [%d,%d,%d] (clips, rows, classes) or [%d,%d], got %s"
                         % (B, Ttot, ncls, B, ncls, shape))
    style = style.to(torch.float32).contiguous()
    if style.numel():
        w = style.double()
        bad_sum = (w.sum(-1) - 1.0).abs().max()
        ok = torch.stack([torch.isfinite(w).all().double(), (w >= 0).all().double(), bad_sum]).tolist()
        if not ok[0]:
            raise ValueError("style weights must be finite")
        if not ok[1]:
            raise ValueError("style weights must be >= 0 (convex mixtures only)")
        if not ok[2] <= 1e-5:
            raise ValueError("every style row must sum to 1 within 1e-5, worst row is off by %g" % ok[2])
    return style


def _controlled(temperature, top_k, noise, want_logp, top_p=1.0, min_p=0.0, want_kept=False, seeds=None):
    """Engine side: validate the controls and the noise source; True when the call leaves the default entry points.
    Sampling takes exactly one of ``noise`` and ``seeds``; greedy decoding needs neither."""
    check_sample_controls(temperature, top_k, top_p, min_p)
    if noise is not None and seeds is not None:
        raise ValueError("give the sampler either noise or seeds, not both")
    if noise is None and seeds is None and float(temperature) > 0:
        raise ValueError("sampling at temperature %g needs the noise tensor or per-clip seeds (only greedy decoding, "
                         "temperature 0, runs without)" % float(temperature))
    return bool(sample_controls(temperature, top_k, want_logp, top_p, min_p)) or bool(want_kept)


def _clip_source(clip, noise, seeds):
    """Engine side of a per-clip call: the noise source rule (exactly one of noise and seeds when any clip samples)."""
    if noise is not None and seeds is not None:
        raise ValueError("give the sampler either noise or seeds, not both")
    if noise is None and seeds is None and (clip["temperature"] > 0).any():
        raise ValueError("clip %d samples at temperature %g: the call needs the noise tensor or per-clip seeds (only a "
                         "batch of greedy clips runs without)" % (int(np.argmax(clip["temperature"] > 0)),
                                                                  float(clip["temperature"].max())))
    return True


def _needs_ctl(top_p, min_p, want_kept):
    """True when a controlled call needs ts_pixelcnn_sample_ctl / ts_body_sample_ctl: top_p, min_p or the keep-set sizes.
    Every other controlled call stays on ts_pixelcnn_sample / ts_body_sample."""
    return float(top_p) < 1.0 or float(min_p) > 0.0 or bool(want_kept)


def _ctl_struct(temperature, top_k, top_p, min_p, logp, kept):
    return _lib.ts_sample_ctl(float(temperature), int(top_k), float(top_p), float(min_p),
                              None if logp is None else logp.data_ptr(), None if kept is None else kept.data_ptr())


class Engine:
    def __init__(self, device=0):
        self.L = _lib.lib()
        h = C.c_void_p()
        dev = device if isinstance(device, int) else torch.device(device).index or 0
        rc = self.L.ts_engine_create(C.byref(h), dev)
        if rc:
            raise RuntimeError("ts_engine_create(%d): %s" % (dev, self.L.ts_last_error(None).decode()))
        self.h = h
        self.host_only = dev < 0
        self.device = torch.device("cuda", dev) if dev >= 0 else torch.device("cpu")
        self.loaded = set()

    def close(self):
        if getattr(self, "h", None):
            self.L.ts_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- helpers ---------------------------------------------------------------------------------
    def _check(self, rc, what):
        if rc:
            raise RuntimeError("%s failed (status %d): %s" % (what, rc, self.L.ts_last_error(self.h).decode()))

    def _s(self):
        return _lib.stream_ptr(self.device)

    def _dev(self, t, dtype):
        return t.to(device=self.device, dtype=dtype).contiguous()

    @property
    def sm_count(self):
        return self.L.ts_engine_sm_count(self.h)

    @property
    def launches(self):
        return int(self.L.ts_launch_count(self.h))

    @property
    def pixelcnn_row_bytes(self):
        return int(self.L.ts_pixelcnn_row_bytes(self.h))

    @property
    def pixelcnn_staged_row_bytes(self):
        return int(self.L.ts_pixelcnn_staged_row_bytes(self.h))

    def pixelcnn_timing(self, enable=True):
        self._check(self.L.ts_pixelcnn_timing(self.h, int(enable)), "ts_pixelcnn_timing")

    def pixelcnn_last_ms(self):
        return float(self.L.ts_pixelcnn_last_ms(self.h))

    def set_tensor_cores(self, enable=True):
        self._check(self.L.ts_set_tensor_cores(self.h, int(enable)), "ts_set_tensor_cores")

    def pixelcnn_trace(self, row):
        """Arm (row >= 0) / disarm (row < 0) the per-stage, per-CTA time stamps of one latent row (debug)."""
        self._check(self.L.ts_pixelcnn_trace(self.h, int(row)), "ts_pixelcnn_trace")

    def pixelcnn_trace_read(self):
        """-> int64 tensor [stages, ctas, 4] (ns): weights ready, left the grid barrier, task done, arrived."""
        import ctypes as C
        n = C.c_int64(0)
        self._check(self.L.ts_pixelcnn_trace_read(self.h, None, C.byref(n)), "ts_pixelcnn_trace_read")
        buf = torch.zeros(n.value, dtype=torch.int64)
        self._check(self.L.ts_pixelcnn_trace_read(self.h, buf.data_ptr(), C.byref(n)), "ts_pixelcnn_trace_read")
        ns, nc = C.c_int(0), C.c_int(0)
        self._check(self.L.ts_pixelcnn_plan_shape(self.h, C.byref(ns), C.byref(nc)), "ts_pixelcnn_plan_shape")
        return buf.view(ns.value, nc.value, 4)

    def set_pixelcnn_fusion(self, on):
        """Plan built by the next load_pixelcnn: 1/True fused 52-stage (default), 0/False plain 84-stage,
        2 fused with vert_to_horiz scheduled in the horizontal pass (experimental)."""
        self._check(self.L.ts_set_pixelcnn_fusion(self.h, int(on)), "ts_set_pixelcnn_fusion")

    def set_pixelcnn_ctas(self, n):
        """Persistent CTAs of the grid-wide sampler plan built by the next load_pixelcnn (0 = one per SM)."""
        self._check(self.L.ts_set_pixelcnn_ctas(self.h, int(n)), "ts_set_pixelcnn_ctas")

    def set_vq_parallel(self, max_batch):
        """body_generate: run the two VQ decoders of batches <= max_batch side by side on two streams (0: one after the other)."""
        self._check(self.L.ts_set_vq_parallel(self.h, int(max_batch)), "ts_set_vq_parallel")

    def set_pixelcnn_mode(self, mode):
        self._check(self.L.ts_set_pixelcnn_mode(self.h, mode), "ts_set_pixelcnn_mode")

    # -- weights ---------------------------------------------------------------------------------
    def load_pixelcnn(self, sd):
        arr, keep = _lib.pack_tensors(sd)
        self._check(self.L.ts_load_pixelcnn(self.h, arr, len(sd)), "ts_load_pixelcnn")
        self.loaded.add("pixelcnn")
        self.pixelcnn_ncls = int(sd["layers.0.class_cond_embedding.weight"].shape[0])   # speaker classes (style=)

    def load_audioenc(self, sd):
        arr, keep = _lib.pack_tensors(sd)
        self._check(self.L.ts_load_audioenc(self.h, arr, len(sd)), "ts_load_audioenc")
        self.loaded.add("audioenc")

    def load_vq(self, which, sd):
        arr, keep = _lib.pack_tensors(sd)
        self._check(self.L.ts_load_vq(self.h, which, arr, len(sd)), "ts_load_vq")
        self.loaded.add("vq%d" % which)

    def load_face(self, sd):
        sd = dict(sd)
        p = "audio_encoder.encoder.pos_conv_embed.conv."
        if p + "weight" not in sd:      # resolve the weight_norm parametrisation (dim=2), old or new names
            if p + "parametrizations.weight.original0" in sd:
                g, v = sd.pop(p + "parametrizations.weight.original0"), sd.pop(p + "parametrizations.weight.original1")
            elif p + "weight_g" in sd and p + "weight_v" in sd:
                g, v = sd.pop(p + "weight_g"), sd.pop(p + "weight_v")
            else:
                raise RuntimeError("ts_load_face: checkpoint tensor '%sweight' (or its weight_norm pair weight_g / weight_v, "
                                   "parametrizations.weight.original0 / original1) missing" % p)
            sd[p + "weight"] = torch._weight_norm(v.float().cpu(), g.float().cpu(), 2)
        arr, keep = _lib.pack_tensors(sd)
        self._check(self.L.ts_load_face(self.h, arr, len(sd)), "ts_load_face")
        self.loaded.add("face")

    # -- modules ---------------------------------------------------------------------------------
    def latent_rows(self, M):
        return self.L.ts_latent_rows(M)

    def mfcc(self, wave, sr):
        """get_mfcc_ta's transform chain on the device: wave [B,N] mono at ``sr`` Hz -> [B,64,M] (30 fps)."""
        wave = self._dev(wave, torch.float32)
        B, N = wave.shape
        M = self.L.ts_mfcc_frames(N, int(sr))
        out = torch.empty(B, 64, M, device=self.device)
        self._check(self.L.ts_mfcc(self.h, _lib.ptr(wave), _lib.ptr(out), B, N, int(sr), self._s()), "ts_mfcc")
        return out

    def silence_mfcc(self, M, B=1):
        """The MFCC [B,64,M] of a silent clip of M frames: ``mfcc`` (the device front end) on a zero waveform at 22 kHz
        whose length gives exactly M frames.  A negative conditioning for audio guidance (``body_generate``)."""
        M = int(M)
        if M < 1:
            raise ValueError("silence_mfcc: M = %d frames" % M)
        n = max(1, (M - 1) * 734)
        while self.L.ts_mfcc_frames(n, 22000) < M:
            n += 1
        while n > 1 and self.L.ts_mfcc_frames(n - 1, 22000) >= M:
            n -= 1
        if self.L.ts_mfcc_frames(n, 22000) != M:
            raise ValueError("silence_mfcc: no waveform length gives %d frames" % M)
        return self.mfcc(torch.zeros(1, n), 22000).repeat(B, 1, 1)

    def audio_encode(self, mfcc):
        """AudioEncoder.forward: [B,64,M] -> [B,256,T]."""
        mfcc = self._dev(mfcc, torch.float32)
        B, _, M = mfcc.shape
        out = torch.empty(B, 256, self.latent_rows(M), device=self.device)
        self._check(self.L.ts_audio_encode(self.h, _lib.ptr(mfcc), _lib.ptr(out), B, M, self._s()), "ts_audio_encode")
        return out

    def sampler_noise(self, seeds, T, T0=0):
        """The Exp(1) values the seeded sampler uses (ts_sampler_noise): seeds [B] (``check_seeds``) -> [2T,B,2048] in the
        layout of ``noise``, block 2(r-T0)+c for the rows r in [T0, T0+T)."""
        if isinstance(T, bool) or int(T) != T or T < 1 or isinstance(T0, bool) or int(T0) != T0 or T0 < 0:
            raise ValueError("sampler_noise: T=%r T0=%r (T >= 1, T0 >= 0)" % (T, T0))
        try:
            n = len(seeds)
        except TypeError:
            raise ValueError("sampler_noise: seeds must be a sequence of integers or an int64 tensor [B], got %r" % (seeds,))
        seeds = self._dev(check_seeds(seeds, n), torch.int64)
        B = seeds.shape[0]
        out = torch.empty(2 * int(T), B, NCODE, device=self.device)
        self._check(self.L.ts_sampler_noise(self.h, _lib.ptr(seeds), _lib.ptr(out), B, int(T), int(T0), self._s()),
                    "ts_sampler_noise")
        return out

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, temperature=1.0, top_k=0,
                          want_logp=False, top_p=1.0, min_p=0.0, want_kept=False, seeds=None, anchors=None, style=None,
                          repetition_penalty=1.0, repetition_window=8, code_bias=None, guidance=None, guide_aud=None,
                          guide_label=None, guide_style=None, want_guide_logp=False):
        """GatedPixelCNN.generate: aud [B,256,T0+T], label [B], noise [2T,B,2048] -> codes [B,T,2]
        (+ logits [2T,B,2048]).  Batches above the 64-sample tile are chunked here.

        Sampling controls (ts_pixelcnn_sample): ``temperature`` (0 = greedy, noise may then be None), ``top_k``
        (0 = off), ``want_logp`` adds logp [B,T,2] = log_softmax(logits)[code] of the untempered model.  The result is
        codes, followed by logits when ``want_logits`` and logp when ``want_logp``.  The defaults call
        ts_pixelcnn_generate.

        ``top_p`` (1 = off) and ``min_p`` (0 = off) truncate the draw further (nucleus / min-p sampling, in the order
        temperature, top_k, top_p, min_p; ts_pixelcnn_sample_ctl); ``want_kept`` appends kept [B,T,2] int32, the number
        of codes each draw chose among.

        ``seeds`` [B] (``check_seeds``) replaces ``noise`` (pass None): seeded sampling, each clip's noise generated in the
        sampler from its own seed and the absolute row of the draw (ts_pixelcnn_sample_seeded; RNG contract in
        include/talkshow_b200.h).  Sampling takes exactly one of the two.

        ``anchors`` [B,T,2] (``check_anchors``: int64 tensor, host or device, or integer numpy array) pins chosen draws:
        a value in [0, 2048) is the code of that draw, -1 samples it as the call without anchors would, with the same
        noise or seeds and controls (ts_pixelcnn_sample_anchored).  With ``pre_latents`` anchor row i is row T0+i.  A pinned
        code conditions later draws only (the prior is causal).  Values are checked (ValueError); for a device tensor that
        costs one synchronisation.  None forwards exactly what the call forwards without it.

        ``style`` (``check_style``: [B,T0+T,ncls] or [B,ncls], float) replaces the speaker label with a per-row convex
        mixture of the prior's speaker embeddings (ts_pixelcnn_sample_styled; rule in include/talkshow_b200.h).  Its rows
        cover every row the network sees, the ``pre_latents`` prefix included; ``label`` is then not read and may be None.
        A one-hot schedule of class s draws what label s draws.  None forwards exactly what the call forwards without it.

        Per-clip controls: ``temperature``, ``top_k``, ``top_p`` and ``min_p`` each take a scalar or one value per clip
        (a length-B sequence, 1-D numpy array or 1-D tensor; ``check_clip_controls``), a scalar among them applying to every
        clip.  Clip b then draws exactly what it draws alone under its own values (ts_pixelcnn_sample_clips), whatever the
        other clips' values; a greedy clip reads no noise.  Sampling takes exactly one of noise and seeds when any clip has
        temperature > 0.  All-scalar calls forward what they forwarded before.

        Logit shaping (ts_pixelcnn_sample_shaped; rule in include/talkshow_b200.h): ``repetition_penalty`` (theta >= 1,
        1 = off) divides a positive logit by theta and multiplies a negative one by it for every code drawn at the same
        column in the clip's previous ``repetition_window`` rows (prefix rows and pinned draws included); ``code_bias``
        (``check_code_bias``: [2,2048] or [B,2,2048], -inf bans a code) is then added.  The controls act on the shaped
        logits; logp stays that of the raw prior.  The penalty and window take a scalar or one value per clip
        (``check_clip_shape``).  Without a bias and with theta 1 everywhere the call forwards what it forwarded before.

        Guided sampling (ts_pixelcnn_sample_guided; rule in include/talkshow_b200.h): ``guidance`` w (``check_guidance``:
        scalar or per clip, in [0, 100], 1 = none) draws every code from g = l_c + (w - 1) (l_c - l_u), l_c the clip's
        logits and l_u those under a negative conditioning: ``guide_aud`` [B,256,T0+T], ``guide_label`` [B] and / or
        ``guide_style`` (as ``style``).  A field not given copies the clip's own; at least one must be given and differ.
        The negative branch is fed the guided codes, so both branches follow the same motion.  The check that the negative
        differs reads no device data: a device tensor counts as the clip's own only when it is the same memory.  Every draw input stays per
        clip; logp is the clip's conditional log p; ``want_guide_logp`` appends the negative branch's log p [B,T,2];
        ``want_logits`` gives the raw logits of both branches, [2T,2B,2048] with clip b's in column 2b.  Each
        launch holds 32 clips (64 branches).  Without ``guidance`` the call forwards what it forwarded before."""
        if guidance is not None:
            return self._guided("pixel", aud, label, noise, T=T, pre_latents=pre_latents, want_logits=want_logits,
                                temperature=temperature, top_k=top_k, want_logp=want_logp, top_p=top_p, min_p=min_p,
                                want_kept=want_kept, seeds=seeds, anchors=anchors, style=style,
                                repetition_penalty=repetition_penalty, repetition_window=repetition_window,
                                code_bias=code_bias, guidance=guidance, guide_cond=guide_aud, guide_label=guide_label,
                                guide_style=guide_style, want_guide_logp=want_guide_logp)
        if guide_aud is not None or guide_label is not None or guide_style is not None or want_guide_logp:
            raise ValueError("pixelcnn_generate: guide_aud / guide_label / guide_style / want_guide_logp need guidance")
        clip = None
        if per_clip(temperature, top_k, top_p, min_p):
            clip = check_clip_controls(temperature, top_k, top_p, min_p, aud.shape[0])
            ctl = _clip_source(clip, noise, seeds)
        else:
            ctl = _controlled(temperature, top_k, noise, want_logp, top_p, min_p, want_kept, seeds)
        shape = check_clip_shape(repetition_penalty, repetition_window, aud.shape[0])
        penalised = bool((shape["repetition_penalty"] != 1.0).any())
        aud = self._dev(aud, torch.float32)
        B = aud.shape[0]
        bias = None if code_bias is None else self._dev(check_code_bias(code_bias, B), torch.float32)
        if label is None and style is None:
            raise ValueError("pixelcnn_generate: label is required without style")
        label = None if label is None else self._dev(label, torch.int64)
        noise = None if noise is None else self._dev(noise, torch.float32)
        seeds = None if seeds is None else self._dev(check_seeds(seeds, B), torch.int64)
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        T = aud.shape[2] - T0 if T is None else T
        anchors = None if anchors is None else self._dev(check_anchors(anchors, B, T), torch.int64)
        style = None if style is None else self._dev(check_style(style, B, T0 + T, self.pixelcnn_ncls), torch.float32)
        if label is not None and label.numel() == 1 and B > 1:
            label = label.expand(B).contiguous()
        pre = None if pre_latents is None else self._dev(pre_latents, torch.int64)
        codes = torch.empty(B, T, 2, dtype=torch.int64, device=self.device)
        logits = torch.empty(2 * T, B, 2048, device=self.device) if want_logits else None
        logp = torch.empty(B, T, 2, device=self.device) if want_logp else None
        kept = torch.empty(B, T, 2, dtype=torch.int32, device=self.device) if want_kept else None
        aud_c = aud.shape[1]
        assert aud_c == 256, "AudioEncoder output has 256 channels"
        for b0 in range(0, B, PIX_TILE):
            b1 = min(B, b0 + PIX_TILE)
            nb = b1 - b0
            full = nb == B
            nz = noise if (full or noise is None) else noise[:, b0:b1].contiguous()
            cz = codes if full else torch.empty(nb, T, 2, dtype=torch.int64, device=self.device)
            lz = logits if (full or logits is None) else torch.empty(2 * T, nb, 2048, device=self.device)
            pz = logp if (full or logp is None) else torch.empty(nb, T, 2, device=self.device)
            kz = kept if (full or kept is None) else torch.empty(nb, T, 2, dtype=torch.int32, device=self.device)
            args = (self.h, _lib.ptr(aud[b0:b1].contiguous()), _lib.ptr(None if label is None else label[b0:b1].contiguous()), _lib.ptr(nz),
                    _lib.ptr(cz), _lib.ptr(lz), nb, T, _lib.ptr(None if pre is None else pre[b0:b1].contiguous()), T0)
            if penalised or bias is not None:
                c = (_ctl_struct(1.0, 0, 1.0, 0.0, pz, kz) if clip is not None
                     else _ctl_struct(temperature, top_k, top_p, min_p, pz, kz))
                args = args[:3] + (_lib.ptr(None if style is None else style[b0:b1]), self.pixelcnn_ncls, _lib.ptr(nz),
                                   _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(None if anchors is None else anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_pixelcnn_sample_shaped(*args, C.byref(c), None if clip is None else clip[b0:b1].ctypes.data,
                                                             shape[b0:b1].ctypes.data if penalised else None,
                                                             _lib.ptr(None if bias is None else bias[b0:b1]), self._s()),
                            "ts_pixelcnn_sample_shaped")
            elif clip is not None:
                c = _ctl_struct(1.0, 0, 1.0, 0.0, pz, kz)      # logp / kept only: the draws' controls are clip[b0:b1]
                args = args[:3] + (_lib.ptr(None if style is None else style[b0:b1]), self.pixelcnn_ncls, _lib.ptr(nz),
                                   _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(None if anchors is None else anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_pixelcnn_sample_clips(*args, C.byref(c), clip[b0:b1].ctypes.data, self._s()),
                            "ts_pixelcnn_sample_clips")
            elif style is not None:
                c = _ctl_struct(temperature, top_k, top_p, min_p, pz, kz) if ctl else None
                args = args[:3] + (_lib.ptr(style[b0:b1]), self.pixelcnn_ncls, _lib.ptr(nz),
                                   _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(None if anchors is None else anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_pixelcnn_sample_styled(*args, None if c is None else C.byref(c), self._s()),
                            "ts_pixelcnn_sample_styled")
            elif anchors is not None:
                c = _ctl_struct(temperature, top_k, top_p, min_p, pz, kz) if ctl else None
                args = args[:3] + (_lib.ptr(nz), _lib.ptr(None if seeds is None else seeds[b0:b1]), _lib.ptr(anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_pixelcnn_sample_anchored(*args, None if c is None else C.byref(c), self._s()),
                            "ts_pixelcnn_sample_anchored")
            elif seeds is not None:
                c = _ctl_struct(temperature, top_k, top_p, min_p, pz, kz) if ctl else None
                args = args[:3] + (_lib.ptr(seeds[b0:b1]),) + args[4:]
                self._check(self.L.ts_pixelcnn_sample_seeded(*args, None if c is None else C.byref(c), self._s()),
                            "ts_pixelcnn_sample_seeded")
            elif ctl and _needs_ctl(top_p, min_p, want_kept):
                c = _ctl_struct(temperature, top_k, top_p, min_p, pz, kz)
                self._check(self.L.ts_pixelcnn_sample_ctl(*args, C.byref(c), self._s()), "ts_pixelcnn_sample_ctl")
            elif ctl:
                self._check(self.L.ts_pixelcnn_sample(*args, float(temperature), int(top_k), _lib.ptr(pz), self._s()),
                            "ts_pixelcnn_sample")
            else:
                self._check(self.L.ts_pixelcnn_generate(*args, self._s()), "ts_pixelcnn_generate")
            if not full:
                codes[b0:b1] = cz
                if logits is not None:
                    logits[:, b0:b1] = lz
                if logp is not None:
                    logp[b0:b1] = pz
                if kept is not None:
                    kept[b0:b1] = kz
        out = (codes,) + ((logits,) if want_logits else ()) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())
        return out if len(out) > 1 else codes

    def pixelcnn_logits(self, aud, label, codes):
        """GatedPixelCNN.forward (teacher forced): -> logits [B,2048,T,2]."""
        aud = self._dev(aud, torch.float32)
        label = self._dev(label, torch.int64)
        codes = self._dev(codes, torch.int64)
        B, _, T = aud.shape
        assert B <= PIX_TILE
        out = torch.empty(B, 2048, T, 2, device=self.device)
        self._check(self.L.ts_pixelcnn_logits(self.h, _lib.ptr(aud), _lib.ptr(label), _lib.ptr(codes), _lib.ptr(out),
                                              B, T, self._s()), "ts_pixelcnn_logits")
        return out

    def pixelcnn_score(self, aud, label, codes, want_logits=False, style=None):
        """Teacher-forced GatedPixelCNN.forward over all rows at once + per-position cross-entropy: aud [B,256,T],
        label [B], codes [B,T,2] -> nll [B,T,2] = -log softmax(logits)[code] (+ logits [B,2048,T,2]).  Any batch size.
        ``style`` ([B,T,ncls] or [B,ncls], ``check_style``): score under a speaker schedule (ts_pixelcnn_score_styled);
        ``label`` is then not read and may be None."""
        aud = self._dev(aud, torch.float32)
        if label is None and style is None:
            raise ValueError("pixelcnn_score: label is required without style")
        label = None if label is None else self._dev(label, torch.int64).reshape(-1)
        codes = self._dev(codes, torch.int64)
        B, _, T = aud.shape
        if label is not None and label.numel() == 1 and B > 1:
            label = label.expand(B).contiguous()
        if aud.shape[1] != 256 or tuple(codes.shape) != (B, T, 2) or (label is not None and label.numel() != B):
            raise ValueError("pixelcnn_score: aud %s, label %s, codes %s (expected [B,256,T], [B], [B,T,2])"
                             % (tuple(aud.shape), tuple(label.shape), tuple(codes.shape)))
        nll = torch.empty(B, T, 2, device=self.device)
        logits = torch.empty(B, 2048, T, 2, device=self.device) if want_logits else None
        if style is not None:
            style = self._dev(check_style(style, B, T, self.pixelcnn_ncls), torch.float32)
            self._check(self.L.ts_pixelcnn_score_styled(self.h, _lib.ptr(aud), _lib.ptr(label), _lib.ptr(style),
                                                        self.pixelcnn_ncls, _lib.ptr(codes), _lib.ptr(nll), _lib.ptr(logits),
                                                        B, T, self._s()), "ts_pixelcnn_score_styled")
            return (nll, logits) if want_logits else nll
        self._check(self.L.ts_pixelcnn_score(self.h, _lib.ptr(aud), _lib.ptr(label), _lib.ptr(codes), _lib.ptr(nll),
                                             _lib.ptr(logits), B, T, self._s()), "ts_pixelcnn_score")
        return (nll, logits) if want_logits else nll

    def vq_dim(self, which):
        """pose channels of the loaded VQ-VAE: 39 / 90 (axis-angle), 78 / 180 (convert_to_6d)."""
        c = int(self.L.ts_vq_dim(self.h, which))
        if c <= 0:
            raise RuntimeError("vq weights %d not loaded" % which)
        return c

    def vq_decode(self, which, idx):
        """VQVAE.decode(latents=idx): [B,T] -> [B,C,4T]."""
        idx = self._dev(idx, torch.int64)
        B, T = idx.shape
        C_ = self.vq_dim(which)
        out = torch.empty(B, C_, 4 * T, device=self.device)
        self._check(self.L.ts_vq_decode(self.h, which, _lib.ptr(idx), _lib.ptr(out), B, T, self._s()), "ts_vq_decode")
        return out

    def vq_encode(self, which, poses, want_e=False):
        """VQVAE.encode: poses [B,F,C] -> idx [B,T] (and e [B,64,T])."""
        poses = self._dev(poses, torch.float32)
        B, F, _ = poses.shape
        T = self.latent_rows(F)
        idx = torch.empty(B, T, dtype=torch.int64, device=self.device)
        e = torch.empty(B, 64, T, device=self.device) if want_e else None
        self._check(self.L.ts_vq_encode(self.h, which, _lib.ptr(poses), _lib.ptr(idx), _lib.ptr(e), B, F, self._s()),
                    "ts_vq_encode")
        return (idx, e) if want_e else idx

    def vq_score(self, which, poses, want_recon=False):
        """Held-out VQ-VAE score (vq_train + get_loss, eval): poses [B,F,C] (C = vq_dim, F % 4 == 0) -> (idx [B,T],
        clip [B,3] float64 = per-clip sums of |recon - gt|, |d recon - d gt| and ||z - e[idx]||^2, recon [B,F,C] or None).
        idx equals vq_encode's, recon equals vq_decode(idx) transposed."""
        poses = self._dev(poses, torch.float32)
        C_ = self.vq_dim(which)
        if poses.dim() != 3 or poses.shape[2] != C_ or poses.shape[0] < 1 or poses.shape[1] < 4 or poses.shape[1] % 4:
            raise ValueError("vq_score: poses %s (expected [B,F,%d] with F a positive multiple of 4)"
                             % (tuple(poses.shape), C_))
        B, F_, _ = poses.shape
        idx = torch.empty(B, F_ // 4, dtype=torch.int64, device=self.device)
        clip = torch.empty(B, 3, dtype=torch.float64, device=self.device)
        recon = torch.empty(B, F_, C_, device=self.device) if want_recon else None
        self._check(self.L.ts_vq_score(self.h, which, _lib.ptr(poses), _lib.ptr(idx), _lib.ptr(recon), _lib.ptr(clip), B, F_,
                                       self._s()), "ts_vq_score")
        return idx, clip, recon

    def face_score(self, wave, id_onehot, gt, want_pred=False):
        """Held-out face score (__call__ + get_loss, eval, frame = F): wave [B,N], id [B,4], gt [B,F,Cgt] (pose columns,
        then the 100 expression columns) -> (clip [B,2] float64 = per-clip sums of |pred[..,:6] - gt[..,:6]| and
        (pred[..,-100:] - gt[..,-100:])^2, pred [B,F,face_dim] or None).  pred equals face_forward(wave, id, F)."""
        wave = self._dev(wave, torch.float32)
        gt = self._dev(gt, torch.float32)
        D = self.face_dim
        if wave.dim() != 2 or gt.dim() != 3 or gt.shape[0] != wave.shape[0] or gt.shape[2] < 100 or gt.shape[1] < 1:
            raise ValueError("face_score: wave %s, gt %s (expected [B,N] and [B,F,C] with C >= 100)"
                             % (tuple(wave.shape), tuple(gt.shape)))
        B, N = wave.shape
        F_ = gt.shape[1]
        if D == 106:
            idv = None
        else:
            idv = self._dev(id_onehot, torch.float32)
            if idv.shape[0] == 1 and B > 1:
                idv = idv.expand(B, -1).contiguous()
            if tuple(idv.shape) != (B, 4):
                raise ValueError("face_score: id %s (expected [B,4])" % (tuple(idv.shape),))
        clip = torch.empty(B, 2, dtype=torch.float64, device=self.device)
        pred = torch.empty(B, F_, D or 103, device=self.device) if want_pred else None
        self._check(self.L.ts_face_score(self.h, _lib.ptr(wave), _lib.ptr(idv), _lib.ptr(gt), gt.shape[2], _lib.ptr(pred),
                                         _lib.ptr(clip), B, N, F_, self._s()), "ts_face_score")
        return clip, pred

    @property
    def face_dim(self):
        """output columns of the loaded face net: 103 (3-D jaw), 106 (6-D jaw, identity-free net); 0 when none is loaded."""
        return int(self.L.ts_face_dim(self.h))

    def face_forward(self, wave, id_onehot, frame):
        """s2g_face.Generator.forward: wave [B,N], id [B,4] -> [B,frame,face_dim].  The identity-free (6-D) net ignores id."""
        wave = self._dev(wave, torch.float32)
        B, N = wave.shape
        D = self.face_dim
        if D == 106:
            idv = None
        else:
            idv = self._dev(id_onehot, torch.float32)
            if idv.shape[0] == 1 and B > 1:
                idv = idv.expand(B, -1).contiguous()
        out = torch.empty(B, frame, D or 103, device=self.device)
        self._check(self.L.ts_face_forward(self.h, _lib.ptr(wave), _lib.ptr(idv), _lib.ptr(out), B, N, frame,
                                           self._s()), "ts_face_forward")
        return out

    def body_generate(self, mfcc, label, noise, want_codes=True, temperature=1.0, top_k=0, want_logp=False, top_p=1.0,
                      min_p=0.0, want_kept=False, seeds=None, anchors=None, style=None, repetition_penalty=1.0,
                      repetition_window=8, code_bias=None, guidance=None, guide_mfcc=None, guide_label=None,
                      guide_style=None, want_guide_logp=False):
        """fused s2g_body_pixel core: mfcc [B,64,M] -> (codes [B,T,2], poses [B,4T,C]), C = 129 (258 for 6-D).
        Sampling controls as in ``pixelcnn_generate`` (ts_body_sample, ts_body_sample_ctl); ``want_logp`` appends logp
        [B,T,2], ``want_kept`` then kept [B,T,2] int32.  ``seeds`` [B] in place of ``noise``: seeded sampling
        (ts_body_sample_seeded), as in ``pixelcnn_generate``.  ``anchors`` [B,T,2] pins draws as in ``pixelcnn_generate``
        (ts_body_sample_anchored; one synchronisation for a device tensor); the poses decode the resulting codes.
        ``style`` [B,T,ncls] or [B,ncls]: a speaker schedule as in ``pixelcnn_generate`` (ts_body_sample_styled; label
        may then be None).  Per-clip ``temperature`` / ``top_k`` / ``top_p`` / ``min_p`` as in ``pixelcnn_generate``
        (ts_body_sample_clips); each clip's poses decode its own codes.  ``repetition_penalty`` / ``repetition_window`` /
        ``code_bias``: logit shaping as in ``pixelcnn_generate`` (ts_body_sample_shaped).  ``guidance`` with ``guide_mfcc``
        [B,64,M] / ``guide_label`` / ``guide_style``: guided sampling as in ``pixelcnn_generate`` (ts_body_sample_guided);
        codes and poses are the clips' (the negative branches are not decoded), ``want_guide_logp`` appends the negative
        branches' log p [B,T,2]."""
        if guidance is not None:
            return self._guided("body", mfcc, label, noise, want_codes=want_codes, temperature=temperature, top_k=top_k,
                                want_logp=want_logp, top_p=top_p, min_p=min_p, want_kept=want_kept, seeds=seeds,
                                anchors=anchors, style=style, repetition_penalty=repetition_penalty,
                                repetition_window=repetition_window, code_bias=code_bias, guidance=guidance,
                                guide_cond=guide_mfcc, guide_label=guide_label, guide_style=guide_style,
                                want_guide_logp=want_guide_logp)
        if guide_mfcc is not None or guide_label is not None or guide_style is not None or want_guide_logp:
            raise ValueError("body_generate: guide_mfcc / guide_label / guide_style / want_guide_logp need guidance")
        clip = None
        if per_clip(temperature, top_k, top_p, min_p):
            clip = check_clip_controls(temperature, top_k, top_p, min_p, mfcc.shape[0])
            ctl = _clip_source(clip, noise, seeds)
        else:
            ctl = _controlled(temperature, top_k, noise, want_logp, top_p, min_p, want_kept, seeds)
        shape = check_clip_shape(repetition_penalty, repetition_window, mfcc.shape[0])
        penalised = bool((shape["repetition_penalty"] != 1.0).any())
        bias = None if code_bias is None else self._dev(check_code_bias(code_bias, mfcc.shape[0]), torch.float32)
        mfcc = self._dev(mfcc, torch.float32)
        if label is None and style is None:
            raise ValueError("body_generate: label is required without style")
        label = None if label is None else self._dev(label, torch.int64)
        noise = None if noise is None else self._dev(noise, torch.float32)
        B, _, M = mfcc.shape
        seeds = None if seeds is None else self._dev(check_seeds(seeds, B), torch.int64)
        if label is not None and label.numel() == 1 and B > 1:
            label = label.expand(B).contiguous()
        T = self.latent_rows(M)
        anchors = None if anchors is None else self._dev(check_anchors(anchors, B, T), torch.int64)
        style = None if style is None else self._dev(check_style(style, B, T, self.pixelcnn_ncls), torch.float32)
        codes = torch.empty(B, T, 2, dtype=torch.int64, device=self.device) if want_codes else None
        poses = torch.empty(B, 4 * T, self.vq_dim(0) + self.vq_dim(1), device=self.device)
        logp = torch.empty(B, T, 2, device=self.device) if want_logp else None
        kept = torch.empty(B, T, 2, dtype=torch.int32, device=self.device) if want_kept else None
        for b0 in range(0, B, PIX_TILE):
            b1 = min(B, b0 + PIX_TILE)
            full = (b1 - b0) == B
            nz = noise if (full or noise is None) else noise[:, b0:b1].contiguous()
            args = (self.h, _lib.ptr(mfcc[b0:b1]), _lib.ptr(None if label is None else label[b0:b1]), _lib.ptr(nz),
                    _lib.ptr(None if codes is None else codes[b0:b1]), _lib.ptr(poses[b0:b1]), b1 - b0, M)
            if penalised or bias is not None:
                lz, kz = None if logp is None else logp[b0:b1], None if kept is None else kept[b0:b1]
                c = _ctl_struct(1.0, 0, 1.0, 0.0, lz, kz) if clip is not None else _ctl_struct(temperature, top_k, top_p, min_p, lz, kz)
                args = args[:3] + (_lib.ptr(None if style is None else style[b0:b1]), self.pixelcnn_ncls, _lib.ptr(nz),
                                   _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(None if anchors is None else anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_body_sample_shaped(*args, C.byref(c), None if clip is None else clip[b0:b1].ctypes.data,
                                                         shape[b0:b1].ctypes.data if penalised else None,
                                                         _lib.ptr(None if bias is None else bias[b0:b1]), self._s()),
                            "ts_body_sample_shaped")
            elif clip is not None:
                c = _ctl_struct(1.0, 0, 1.0, 0.0, None if logp is None else logp[b0:b1], None if kept is None else kept[b0:b1])
                args = args[:3] + (_lib.ptr(None if style is None else style[b0:b1]), self.pixelcnn_ncls, _lib.ptr(nz),
                                   _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(None if anchors is None else anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_body_sample_clips(*args, C.byref(c), clip[b0:b1].ctypes.data, self._s()),
                            "ts_body_sample_clips")
            elif style is not None:
                c = None
                if ctl:
                    c = _ctl_struct(temperature, top_k, top_p, min_p, None if logp is None else logp[b0:b1],
                                    None if kept is None else kept[b0:b1])
                args = args[:3] + (_lib.ptr(style[b0:b1]), self.pixelcnn_ncls, _lib.ptr(nz),
                                   _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(None if anchors is None else anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_body_sample_styled(*args, None if c is None else C.byref(c), self._s()),
                            "ts_body_sample_styled")
            elif anchors is not None:
                c = None
                if ctl:
                    c = _ctl_struct(temperature, top_k, top_p, min_p, None if logp is None else logp[b0:b1],
                                    None if kept is None else kept[b0:b1])
                args = args[:3] + (_lib.ptr(nz), _lib.ptr(None if seeds is None else seeds[b0:b1]),
                                   _lib.ptr(anchors[b0:b1])) + args[4:]
                self._check(self.L.ts_body_sample_anchored(*args, None if c is None else C.byref(c), self._s()),
                            "ts_body_sample_anchored")
            elif seeds is not None:
                c = None
                if ctl:
                    c = _ctl_struct(temperature, top_k, top_p, min_p, None if logp is None else logp[b0:b1],
                                    None if kept is None else kept[b0:b1])
                args = args[:3] + (_lib.ptr(seeds[b0:b1]),) + args[4:]
                self._check(self.L.ts_body_sample_seeded(*args, None if c is None else C.byref(c), self._s()),
                            "ts_body_sample_seeded")
            elif ctl and _needs_ctl(top_p, min_p, want_kept):
                c = _ctl_struct(temperature, top_k, top_p, min_p, None if logp is None else logp[b0:b1],
                                None if kept is None else kept[b0:b1])
                self._check(self.L.ts_body_sample_ctl(*args, C.byref(c), self._s()), "ts_body_sample_ctl")
            elif ctl:
                self._check(self.L.ts_body_sample(*args, float(temperature), int(top_k),
                                                  _lib.ptr(None if logp is None else logp[b0:b1]), self._s()),
                            "ts_body_sample")
            else:
                self._check(self.L.ts_body_generate(*args, self._s()), "ts_body_generate")
        return (codes, poses) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())

    def _guided(self, kind, cond, label, noise, T=None, pre_latents=None, want_logits=False, want_codes=True,
                temperature=1.0, top_k=0, want_logp=False, top_p=1.0, min_p=0.0, want_kept=False, seeds=None, anchors=None,
                style=None, repetition_penalty=1.0, repetition_window=8, code_bias=None, guidance=None, guide_cond=None,
                guide_label=None, guide_style=None, want_guide_logp=False):
        """The guided calls of ``pixelcnn_generate`` (kind "pixel", cond = aud) and ``body_generate`` (kind "body", cond =
        mfcc): B clips -> 2B interleaved branches (2b the clip, 2b + 1 its negative conditioning), every draw input per
        clip, GUIDE_PAIRS clips per launch."""
        who = "pixelcnn_generate" if kind == "pixel" else "body_generate"
        B = cond.shape[0]
        w = check_guidance(guidance, B)
        if guide_cond is None and guide_label is None and guide_style is None:
            raise ValueError("%s: guidance needs a negative conditioning (guide_%s, guide_label or guide_style)"
                             % (who, "aud" if kind == "pixel" else "mfcc"))
        clip = None
        if per_clip(temperature, top_k, top_p, min_p):
            clip = check_clip_controls(temperature, top_k, top_p, min_p, B)
            _clip_source(clip, noise, seeds)
        else:
            _controlled(temperature, top_k, noise, want_logp, top_p, min_p, want_kept, seeds)
        shape = check_clip_shape(repetition_penalty, repetition_window, B)
        penalised = bool((shape["repetition_penalty"] != 1.0).any())
        bias = None if code_bias is None else self._dev(check_code_bias(code_bias, B), torch.float32)
        # the negative must differ from the clip in some field (checked on the inputs as given: no synchronisation)
        if guide_label is not None:
            same_class = label is not None and style is None and guide_style is None and _same_input(label, guide_label)
        elif guide_style is not None:
            same_class = style is not None and _same_input(style, guide_style)
        else:
            same_class = True
        if same_class and (guide_cond is None or _same_input(cond, guide_cond)):
            raise ValueError("%s: the negative conditioning equals the clips' own: guidance would change nothing" % who)
        cond = self._dev(cond, torch.float32)
        gcond = cond if guide_cond is None else self._dev(guide_cond, torch.float32)
        if tuple(gcond.shape) != tuple(cond.shape):
            raise ValueError("%s: the negative conditioning has shape %s, the clips %s"
                             % (who, tuple(gcond.shape), tuple(cond.shape)))
        if label is None and style is None:
            raise ValueError("%s: label is required without style" % who)
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        if kind == "pixel":
            T = cond.shape[2] - T0 if T is None else T
        else:
            T = self.latent_rows(cond.shape[2])
        ncls = self.pixelcnn_ncls

        def labels(v):
            v = self._dev(v if torch.is_tensor(v) else torch.as_tensor(v), torch.int64).reshape(-1)
            return v.expand(B).contiguous() if v.numel() == 1 and B > 1 else v

        def one_hot(v):   # a label as its one-hot schedule, which draws what the label draws (ts_pixelcnn_sample_styled)
            return torch.nn.functional.one_hot(v.clamp(0, ncls - 1), ncls).to(torch.float32)

        label = None if label is None else labels(label)
        glabel = None if guide_label is None else labels(guide_label)
        style = None if style is None else self._dev(check_style(style, B, T0 + T, ncls), torch.float32)
        gstyle = None if guide_style is None else self._dev(check_style(guide_style, B, T0 + T, ncls), torch.float32)
        if style is None and gstyle is None:   # labels on both branches
            label2, style2 = _interleave(label, label if glabel is None else glabel), None
        else:                                  # a schedule on either side: both branches as schedules
            cs = style if style is not None else one_hot(label)[:, None, :].expand(B, T0 + T, ncls)
            gs = gstyle if gstyle is not None else (one_hot(glabel)[:, None, :].expand(B, T0 + T, ncls)
                                                    if glabel is not None else cs)
            label2, style2 = None, _interleave(cs, gs)
        cond2 = _interleave(cond, gcond)
        noise = None if noise is None else self._dev(noise, torch.float32)
        seeds = None if seeds is None else self._dev(check_seeds(seeds, B), torch.int64)
        anchors = None if anchors is None else self._dev(check_anchors(anchors, B, T), torch.int64)
        pre = None if pre_latents is None else self._dev(pre_latents, torch.int64)
        idx = torch.empty(2 * B, T, 2, dtype=torch.int64, device=self.device) if (kind == "pixel" or want_codes) else None
        logits = torch.empty(2 * T, 2 * B, 2048, device=self.device) if want_logits else None
        lp = torch.empty(2 * B, T, 2, device=self.device) if (want_logp or want_guide_logp) else None
        kept = torch.empty(2 * B, T, 2, dtype=torch.int32, device=self.device) if want_kept else None
        poses = torch.empty(B, 4 * T, self.vq_dim(0) + self.vq_dim(1), device=self.device) if kind == "body" else None
        sl = lambda t, a, b: None if t is None else t[a:b].contiguous()
        for b0 in range(0, B, GUIDE_PAIRS):
            b1 = min(B, b0 + GUIDE_PAIRS)
            nb, r0, r1 = b1 - b0, 2 * b0, 2 * b1
            nz = noise if (noise is None or nb == B) else noise[:, b0:b1].contiguous()
            lz = None if logits is None else (logits if nb == B else torch.empty(2 * T, 2 * nb, 2048, device=self.device))
            c = (_ctl_struct(1.0, 0, 1.0, 0.0, sl(lp, r0, r1), sl(kept, r0, r1)) if clip is not None
                 else _ctl_struct(temperature, top_k, top_p, min_p, sl(lp, r0, r1), sl(kept, r0, r1)))
            head = (self.h, _lib.ptr(cond2[r0:r1]), _lib.ptr(sl(label2, r0, r1)), _lib.ptr(sl(style2, r0, r1)), ncls,
                    _lib.ptr(nz), _lib.ptr(sl(seeds, b0, b1)), _lib.ptr(sl(anchors, b0, b1)))
            tail = (C.byref(c), None if clip is None else clip[b0:b1].ctypes.data,
                    shape[b0:b1].ctypes.data if penalised else None, _lib.ptr(sl(bias, b0, b1)), w[b0:b1].ctypes.data,
                    self._s())
            if kind == "pixel":
                self._check(self.L.ts_pixelcnn_sample_guided(*head, _lib.ptr(idx[r0:r1]), _lib.ptr(lz), nb, T,
                                                             _lib.ptr(sl(pre, b0, b1)), T0, *tail), "ts_pixelcnn_sample_guided")
            else:
                self._check(self.L.ts_body_sample_guided(*head, _lib.ptr(None if idx is None else idx[r0:r1]),
                                                         _lib.ptr(poses[b0:b1]), nb, cond.shape[2], *tail),
                            "ts_body_sample_guided")
            if lz is not None and nb != B:
                logits[:, r0:r1] = lz
        codes = None if idx is None else idx[0::2].contiguous()
        extra = (((lp[0::2].contiguous(),) if want_logp else ()) + ((kept[0::2].contiguous(),) if want_kept else ())
                 + ((lp[1::2].contiguous(),) if want_guide_logp else ()))
        if kind == "body":
            return (codes, poses) + extra
        out = (codes,) + ((logits,) if want_logits else ()) + extra
        return out if len(out) > 1 else codes

    # -- the single collective of the path, inside the library (ts_allgather over a dlopen'ed NCCL) ----------------
    @staticmethod
    def _libnccl_path():
        import glob
        import os

        base = os.path.dirname(os.path.dirname(torch.__file__))
        hits = glob.glob(os.path.join(base, "nvidia", "nccl", "lib", "libnccl.so*"))
        return (hits[0] if hits else "libnccl.so.2").encode()

    def nccl_init(self, rank, world, group=None):
        """Create this engine's NCCL communicator.  The 128-byte unique id is made on rank 0 and broadcast with
        torch.distributed (any backend: it is 128 bytes of host data), every rank then joins."""
        import torch.distributed as dist

        path = self._libnccl_path()
        buf = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            self._check(self.L.ts_nccl_unique_id(self.h, path, buf.data_ptr()), "ts_nccl_unique_id")
        if world > 1:
            obj = [buf.numpy().tobytes()]
            dist.broadcast_object_list(obj, src=0, group=group)
            buf = torch.frombuffer(bytearray(obj[0]), dtype=torch.uint8).clone()
        self._check(self.L.ts_nccl_init(self.h, path, buf.data_ptr(), rank, world), "ts_nccl_init")
        self.nccl_world = world
        return self

    def allgather(self, local):
        """local [n, ...] fp32 (same shape on every rank) -> [world * n, ...] through ts_allgather (NCCL, current stream)."""
        local = self._dev(local, torch.float32)
        world = getattr(self, "nccl_world", 0)
        if not world:
            raise RuntimeError("Engine.nccl_init was not called")
        out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), device=self.device)
        self._check(self.L.ts_allgather(self.h, _lib.ptr(local), _lib.ptr(out), local.numel(), self._s()), "ts_allgather")
        return out

    def rot6d_to_axis_angle(self, d6):
        """matrix_to_axis_angle(rotation_6d_to_matrix(d6)) (rotation_conversion.py:512-533,433-447): [...,6] -> [...,3]."""
        d6 = self._dev(d6, torch.float32)
        if d6.shape[-1] != 6:
            raise ValueError("rot6d_to_axis_angle: last dim must be 6, got %s" % (tuple(d6.shape),))
        out = torch.empty(d6.shape[:-1] + (3,), device=self.device)
        self._check(self.L.ts_rot6d_to_axis_angle(self.h, _lib.ptr(d6), _lib.ptr(out), d6.numel() // 6, self._s()),
                    "ts_rot6d_to_axis_angle")
        return out

    def assemble_pose(self, face, body, stand=False):
        """demo.py:182-229 + part2full: face [B,Ff,103], body [B,Fb,129] -> [B,Ff,265]; or, for convert_to_6d outputs,
        face [B,Ff,106], body [B,Fb,258] (6-D jaw / joints converted to axis-angle in the same kernel) -> [B,Ff,265]."""
        face = self._dev(face, torch.float32)
        body = self._dev(body, torch.float32)
        if face.dim() != 3 or body.dim() != 3 or body.shape[0] != face.shape[0]:
            raise ValueError("assemble_pose: face %s, body %s (expected [B,Ff,C] and [B,Fb,C])"
                             % (tuple(face.shape), tuple(body.shape)))
        dims = (face.shape[2], body.shape[2])
        if dims == (103, 129):
            fn, name = self.L.ts_assemble_pose, "ts_assemble_pose"
        elif dims == (106, 258):
            fn, name = self.L.ts_assemble_pose6d, "ts_assemble_pose6d"
        else:
            raise ValueError("assemble_pose: face / body columns %s: expected (103, 129) or, 6-D, (106, 258)" % (dims,))
        B, Ff, _ = face.shape
        out = torch.empty(B, Ff, 265, device=self.device)
        self._check(fn(self.h, _lib.ptr(face), _lib.ptr(body), _lib.ptr(out), B, Ff, body.shape[1], int(stand), self._s()), name)
        return out
