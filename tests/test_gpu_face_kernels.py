"""GPU (-m gpu): the face regressor's two hand-written HMMA kernels on their own -- the self-attention (csrc/face.cu:
attention_mma16p_kernel for clips of at most 384 frames, attention_mma16t_kernel beyond, and the three older kernels
TS_ATT_MMA selects) through ts_debug_attention, and the grouped positional conv (posconv_mma_kernel, and the FFMA GEMM it
falls back to with the tensor cores off) through ts_debug_posconv.  Both entries stage the data as the face forward
does and call the chosen kernel directly.  Every result is compared with a float64 evaluation on the GPU of the same
fp32 inputs: softmax(q k^T / 8) v per head, and the grouped conv1d + bias + erf-GELU.

Attention bar, per element (o = sum_j p_j v_j / sum_j p_j, A = sum_j p_j |v_j| / sum_j p_j with the exact p):
  * scores s_j = (q / 8) . k_j.  fp16 split (kernels 2, 3, 4): each operand to 2^-22 while its low plane is normal, the
    dropped lo*lo product below 2^-22 -- 3 * 2^-22 per product -- and 4 k16-steps x 3 products = 12 truncating MMAs per
    score at 2^-22 each (the dense tests' per-MMA term): 15 * 2^-22 * S_j, S_j = sum_d |q_d / 8| |k_jd|.  Below the
    normal range of the low plane the split leaves an absolute 2^-25 per operand: + 2^-25 (sum |q / 8| + sum |k_j|).
    tf32 (kernel 1): 3 * 2^-20 + 8 k8-steps x 3 = 24 MMAs.  FFMA (kernel 0): a 64-long fp32 FMA chain, 64 * 2^-24.
    Subtracting the running max rounds: + 2^-23 max_j |s_j|.  Call the per-row maximum over j of all this ds.
  * the score error carried through the softmax: |do| <= (exp(2 ds) - 1) max_j |v_j| (2 ds max|v| to first order).
  * P V.  p_j = expf(s_j - m) (2 ulp) in numerator and denominator: 2^-21 A.  P is scaled by 2^10 before the split, so its
    low plane stays normal down to p = 2^-13 and below that pays 2^-25 / 2^10 per key: 2^-35 sum_j |v_j| absolute (the row
    sum is >= 1).  v's split: 3 * 2^-22 A and 2^-25 absolute.  MMA chain: kernels 3 and 4 accumulate each 64-key block
    into a fresh fragment (4 k16-steps x 3 = 12 truncating MMAs, 12 * 2^-22 A) added to the output with round-to-nearest
    adds (nb * 2^-24 A, nb = ceil(T / 64) blocks); kernel 2 chains all 12 nb MMAs (12 nb * 2^-22 A), kernel 1 all 24 nb
    (24 nb * 2^-22 A), kernel 0 is a T-long FMA chain (T * 2^-24 A).
  * the row sum (T / 8 adds per lane, a 4-lane tree), the rescales by exp(m_old - m_new) and the final 1 / (1024 l)
    and product: (T / 8 + 4 nb + 16) * 2^-24 A.
An unmasked pad key, a wrong key / value row, a lost 16-key step or chunk, or a dropped hi*lo product (2^-12 of each
product) each move the error by orders of magnitude over these bars.

Positional conv bar, per element (S = sum |x||w| over the 128-tap window of the group, K = 6144): the fp16 split's
3 * 2^-22 S; 4 taps x 3 channel steps x 3 products = 36 truncating MMAs per 4-tap chunk into fresh accumulators,
36 * 2^-22 S, the 32 chunks added round-to-nearest, 32 * 2^-24 S; the absolute underflow term 2^-25 (sum|w| +
sum|x| / 2^shift) with the weights scaled by 2^shift (split16_shift); FFMA (mode 0): K * 2^-24 S.  Epilogue (unscale,
bias): 2^-22 (S + |bias|); the GELU's slope <= 1.13 multiplies all of it and its own fp32 evaluation adds 2^-21 |z|.

Statistical bar: the RMS over the outputs of |error| / A (attention) or |error| / S (posconv) is pinned per kernel at
4x the largest value measured over the cases below on one H100 80GB HBM3 (700 W power limit); see RMS_BAR.  Cases
whose error is dominated by an absolute underflow term (magnitudes of 1e-6, and q scaled down to 1e-5 against keys of
6e4) are checked against the per-element bar only.  Every case prints its statistics ("att ..." / "posconv ..." lines,
pytest -s).

Exact checks: two calls give the same bits; an item gives the same bits alone as inside a batch of 7; the output planes
(fp16: h = fp16(o), l = fp16(o - h); 3xTF32: hi has its 13 low bits clear and hi + lo is the plain output); outputs
are finite with 64 NaN rows after the last item's qkv (ts_debug_attention stages them) and every output element is
written; attention_mma16t_kernel gives the same bits for every chunk of 64 .. 384 keys, and attention_mma16p_kernel and
attention_mma16t_kernel give the same bits at every T <= 384 (each 64-key block is processed the same way whatever the
staging); the face forward's choice is the resident kernel at 384 frames and the tiled one at 385; a one-hot input row
reproduces the tap column of its channel, shifted by the pad of 64, in its own group only; the truncation bias on
positive values; requests a kernel cannot run come back as TS_ERR_INVALID without a launch."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

from talkshow_b200 import _lib

pytestmark = pytest.mark.gpu

TS_ERR_INVALID = 1
H, HD = 12, 64
FFMA, TF32, MMA16, MMA16P, MMA16T = 0, 1, 2, 3, 4
KNAME = {-1: "auto", FFMA: "ffma", TF32: "tf32", MMA16: "mma16", MMA16P: "mma16p", MMA16T: "mma16t"}
SENT = 1234.5
SENT16 = 0x5A5A
# RMS of |error| / A (attention) and |error| / S (posconv), 4x the largest value measured on one H100 80GB HBM3
# (700 W power limit), see the module docstring: per kernel on N(0, 1) inputs (largest measured: FFMA 7.9e-8, tf32
# 3.2e-7, mma16 4.5e-7, mma16p / mma16t 1.17e-6, both at T = 1, where every output is one v), per softmax shape over
# both default kernels (sharp 2.57e-6, flat 2.0e-8, dominant first 2.09e-6, dominant last 5.1e-7), per posconv kernel
# (HMMA 2.52e-8, FFMA 2.83e-8)
RMS_BAR = {"att": {FFMA: 4 * 7.91e-8, TF32: 4 * 3.18e-7, MMA16: 4 * 4.52e-7, MMA16P: 4 * 1.17e-6, MMA16T: 4 * 1.17e-6},
           "shape": {"sharp": 4 * 2.57e-6, "flat": 4 * 2.03e-8, "dom0": 4 * 2.09e-6, "domlast": 4 * 5.05e-7},
           "pc": {6: 4 * 2.52e-8, 0: 4 * 2.83e-8}}
# mean signed error / |o| of the default kernels at T = 384 on positive v with flat-ish scores (test_truncation_bias):
# -2.45e-7 measured for both (H100 80GB HBM3, 700 W)
BIAS_BAR = 2 * 2.45e-7


class DebugAtt(C.Structure):
    _fields_ = [(f, C.c_int32) for f in ("kernel", "B", "T", "chunk", "out_format")]


@pytest.fixture(scope="module")
def eng():
    from talkshow_b200.engine import Engine

    torch.set_grad_enabled(False)
    e = Engine(0)
    yield e
    torch.cuda.synchronize()
    e.close()


# ---- attention ---------------------------------------------------------------------------------------------------------
def make_qkv(B, T, seed, shape="prod"):
    """[B,T,2304] fp32 on the GPU: q, k, v ~ N(0, 1) (score std 1) reshaped by `shape`."""
    gen = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, T, H * HD, generator=gen) for _ in range(3))
    if shape == "sharp":                      # scores std 8: nearly one-hot rows
        q = q * 8
    elif shape == "flat":                     # every score 0: o = mean of the T real values exactly
        q = torch.zeros_like(q)
    elif shape in ("dom0", "domlast"):        # one key far above the others for every query of every head
        j = 0 if shape == "dom0" else T - 1
        q[:, :, ::HD] += 4
        k[:, j, ::HD] = 32
    elif shape == "mag6e4":                   # k, v up to 6e4; q scaled to keep the scores O(1): |q / 8| ~ 1e-5
        def lu(lo, hi):
            mag = torch.exp(torch.empty(B, T, H * HD).uniform_(math.log(lo), math.log(hi), generator=gen))
            return torch.where(torch.rand(B, T, H * HD, generator=gen) < 0.5, -mag, mag)
        k, v = lu(1e2, 6e4), lu(1e2, 6e4)
        q = q / float(k.pow(2).mean().sqrt())
    elif shape == "mag1e-6":
        q, k, v = q * 1e-6, k * 1e-6, v * 1e-6
    elif shape == "posv":                     # positive values, flat-ish scores: the truncation bias shows
        q = q * 0.25
        v = torch.rand(B, T, H * HD, generator=gen) * 0.5 + 0.5
    return torch.cat([q, k, v], 2).contiguous().cuda()


def att_call(e, kernel, qkv, fmt=0, chunk=0, out=None, hi=None, lo=None):
    """-> (status, out, plane_hi, plane_lo, launches issued); buffers start as sentinels unless given."""
    B, T = qkv.shape[:2]
    if out is None:
        out = torch.full((B, T, H * HD), SENT, device="cuda")
    if hi is None and fmt:
        hi = (torch.full((B, T, H * HD), SENT16, dtype=torch.int16, device="cuda") if fmt == 2
              else torch.full((B, T, H * HD), SENT, device="cuda"))
        lo = hi.clone()
    a = DebugAtt(kernel, B, T, chunk, fmt)
    n0 = e.launches
    rc = e.L.ts_debug_attention(e.h, C.byref(a), _lib.ptr(qkv), _lib.ptr(out if fmt != 1 else None), _lib.ptr(hi),
                                _lib.ptr(lo), e._s())
    torch.cuda.synchronize()
    return rc, out, hi, lo, e.launches - n0


def att_reference(qkv):
    """float64 per item: o [B,T,768], A = sum p|v| / sum p, the per-row score terms S_max = max_j (S_j + 2^-25 sum|k_j|)
    + 2^-25 sum|q / 8| (fp16 kernels' form, split below), smax = max_j |s_j|, vmax and vsum = max / sum over j of |v|."""
    B, T, _ = qkv.shape
    out = {n: [] for n in ("o", "A", "Sq", "Sa", "smax", "vmax", "vsum")}
    for b in range(B):
        x = qkv[b].double().view(T, 3, H, HD).permute(1, 2, 0, 3)          # [3, H, T, HD]
        q, k, v = x[0] / 8, x[1], x[2]
        s = q @ k.transpose(1, 2)                                          # [H, T, T]
        p = torch.softmax(s, -1)
        out["o"].append((p @ v).transpose(0, 1).reshape(T, H * HD))
        out["A"].append((p @ v.abs()).transpose(0, 1).reshape(T, H * HD))
        S = q.abs() @ k.abs().transpose(1, 2)
        out["Sq"].append(S.amax(-1))                                       # [H, T]: max_j S_j
        ua = 2.0 ** -25 * (q.abs().sum(-1, keepdim=True) + k.abs().sum(-1).unsqueeze(1))
        out["Sa"].append((15 * 2.0 ** -22 * S + ua).amax(-1))               # the fp16 kernels' whole score term
        out["smax"].append(s.abs().amax(-1))
        out["vmax"].append(v.abs().amax(1))                                # [H, HD]
        out["vsum"].append(v.abs().sum(1))
    return {n: torch.stack(t) for n, t in out.items()}


def att_tol(kernel, T, ref):
    """Per-element bar [B,T,768] of `kernel` (see the module docstring)."""
    nb = -(-T // 64)
    B = ref["o"].shape[0]
    if kernel in (MMA16, MMA16P, MMA16T):
        ds = ref["Sa"]
    elif kernel == TF32:
        ds = (3 * 2.0 ** -20 + 24 * 2.0 ** -22) * ref["Sq"]
    else:
        ds = 65 * 2.0 ** -24 * ref["Sq"]
    ds = ds + 2.0 ** -23 * ref["smax"]                                     # [B, H, T]
    carried = torch.expm1(2 * ds).unsqueeze(-1) * ref["vmax"].unsqueeze(2)  # [B, H, T, HD]
    carried = carried.permute(0, 2, 1, 3).reshape(B, T, H * HD)
    common = 2.0 ** -21 + (T / 8 + 4 * nb + 16) * 2.0 ** -24
    absu = 0.0
    if kernel in (MMA16, MMA16P, MMA16T):
        rel = 3 * 2.0 ** -22 + (12 * 2.0 ** -22 + nb * 2.0 ** -24 if kernel != MMA16 else 12 * nb * 2.0 ** -22)
        absu = (2.0 ** -25 + 2.0 ** -35 * ref["vsum"]).reshape(B, 1, H * HD)
    elif kernel == TF32:
        rel = 3 * 2.0 ** -20 + 24 * nb * 2.0 ** -22
    else:
        rel = T * 2.0 ** -24
    return carried + (rel + common) * ref["A"] + absu


def att_check(kernel, qkv, out, label, rms=True, ref=None, real_kernel=None, shape=None):
    """Accuracy of one call's fp32 output; returns (rms, max) of |error| / A."""
    ref = ref or att_reference(qkv)
    T = qkv.shape[1]
    k = kernel if real_kernel is None else real_kernel
    assert torch.isfinite(out).all(), "%s: non-finite outputs" % label
    err = (out.double() - ref["o"]).abs()
    tol = att_tol(k, T, ref)
    bad = err > tol
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        pytest.fail("%s: %d elements over the bar, first %s: got %.9g ref %.9g tol %.3g A %.3g" % (
            label, int(bad.sum()), i, float(out[i]), float(ref["o"][i]), float(tol[i]), float(ref["A"][i])))
    r = err / ref["A"]
    st_rms, st_max = float(r.pow(2).mean().sqrt()), float(r.max())
    print("att %-34s %-6s B %2d T %4d: rms %.3g max %.3g (err / A), max err / bar %.3g" % (
        label, KNAME[k], qkv.shape[0], T, st_rms, st_max, float((err / tol).max())))
    bar = RMS_BAR["shape"][shape] if shape else RMS_BAR["att"][k]
    if rms:
        assert st_rms <= bar, "%s: RMS err / A %.3g over the bar %.3g" % (label, st_rms, bar)
    return st_rms, st_max


def check_formats(e, kernel, qkv, f0, label, chunk=0):
    """Formats 1 and 2 of the same call against the format-0 output, bit for bit."""
    rc, _, hi, lo, _ = att_call(e, kernel, qkv, fmt=1, chunk=chunk)
    assert rc == 0, label
    assert (hi.view(torch.int32) & 0x1FFF).eq(0).all(), "%s: hi plane with low mantissa bits set" % label
    assert torch.equal(hi + lo, f0), "%s: hi + lo is not the plain output" % label
    if kernel in (FFMA, TF32, MMA16):
        return
    rc, out, h16, l16, _ = att_call(e, kernel, qkv, fmt=2, chunk=chunk)
    assert rc == 0, label
    assert torch.equal(out, f0), "%s: format-2 fp32 output differs from format 0" % label
    on = out.cpu().numpy()
    h = on.astype(np.float16)
    l = (on - h.astype(np.float32)).astype(np.float16)
    assert np.array_equal(h16.cpu().numpy().view(np.uint16), h.view(np.uint16)), label
    assert np.array_equal(l16.cpu().numpy().view(np.uint16), l.view(np.uint16)), label


LENGTHS = [1, 2, 15, 16, 17, 63, 64, 65, 159, 160, 161, 300, 383, 384, 385, 640, 641, 1600, 3100]
LEN_IDS = [(k, T, B) for k in (MMA16P, MMA16T) for T in LENGTHS for B in (1, 3) if k == MMA16T or T <= 384]


@pytest.mark.parametrize("kernel,T,B", LEN_IDS, ids=["%s-T%d-B%d" % (KNAME[k], T, B) for k, T, B in LEN_IDS])
def test_attention_lengths(eng, kernel, T, B):
    """Every row block, query tile, key chunk and dispatch boundary, in all three output formats; at T <= 384 the tiled
    kernel gives the resident kernel's bits."""
    qkv = make_qkv(B, T, seed=zlib.crc32(b"len%d" % T) + B)
    rc, f0, _, _, n = att_call(eng, kernel, qkv)
    assert rc == 0 and n == 1, eng.L.ts_last_error(eng.h)
    att_check(kernel, qkv, f0, "lengths")
    check_formats(eng, kernel, qkv, f0, "T %d" % T)
    if kernel == MMA16T and T <= 384:
        rc, f3, _, _, _ = att_call(eng, MMA16P, qkv)
        assert rc == 0 and torch.equal(f3, f0), "T %d: mma16p and mma16t differ" % T


def test_attention_production_shape(eng):
    """The face forward's 64 clips x 10 s, on the kernel it picks."""
    qkv = make_qkv(64, 300, seed=7)
    rc, f0, _, _, _ = att_call(eng, -1, qkv)
    assert rc == 0
    att_check(-1, qkv, f0, "production 64 x 300", real_kernel=MMA16P)
    check_formats(eng, MMA16P, qkv, f0, "production")


LEGACY = [(k, T) for k in (FFMA, TF32, MMA16) for T in (1, 17, 300, 384)] + [(FFMA, T) for T in (704, 705, 1536, 1537)]


@pytest.mark.parametrize("kernel,T", LEGACY, ids=["%s-T%d" % (KNAME[k], T) for k, T in LEGACY])
def test_attention_legacy(eng, kernel, T):
    """The TS_ATT_MMA kernels in formats 0 and 1, and the FFMA kernel's query-tile switches (64 -> 32 rows at 705,
    32 -> 16 at 1537)."""
    B = 3 if T <= 384 else 1
    qkv = make_qkv(B, T, seed=zlib.crc32(b"legacy%d" % T))
    rc, f0, _, _, n = att_call(eng, kernel, qkv)
    assert rc == 0 and n == 1, eng.L.ts_last_error(eng.h)
    att_check(kernel, qkv, f0, "legacy")
    check_formats(eng, kernel, qkv, f0, "%s T %d" % (KNAME[kernel], T))


SHAPES = ["sharp", "flat", "dom0", "domlast", "mag6e4", "mag1e-6"]
SHAPE_AT = [(MMA16P, 65), (MMA16P, 383), (MMA16T, 641), (MMA16T, 3100)]
SHAPE_IDS = [(s, k, T) for s in SHAPES for k, T in SHAPE_AT]


@pytest.mark.parametrize("shape,kernel,T", SHAPE_IDS, ids=["%s-%s-T%d" % (s, KNAME[k], T) for s, k, T in SHAPE_IDS])
def test_attention_softmax_shapes(eng, shape, kernel, T):
    """Sharp rows, flat rows (o = the mean over the T real keys: a pad key would dilute it by T / Tp), a dominant key
    first or last (the last partial 16-key step and chunk), and magnitudes at the fp16 range limit and in its
    underflow range."""
    qkv = make_qkv(2, T, seed=zlib.crc32(shape.encode()) + T, shape=shape)
    rc, f0, _, _, _ = att_call(eng, kernel, qkv)
    assert rc == 0
    att_check(kernel, qkv, f0, shape, rms=not shape.startswith("mag"), shape=None if shape.startswith("mag") else shape)
    if shape == "flat":
        mean = qkv[:, :, 2 * H * HD:].double().mean(1, keepdim=True)
        assert ((f0.double() - mean).abs() <= 2.0 ** -20 * qkv[:, :, 2 * H * HD:].double().abs().amax(1, keepdim=True)).all()


def test_attention_exact(eng):
    """Same bits on a second call, and for an item alone as inside a batch of 7."""
    for kernel, T in ((MMA16P, 300), (MMA16T, 161), (MMA16T, 641), (TF32, 100), (FFMA, 100), (MMA16, 100)):
        qkv = make_qkv(7, T, seed=40 + T)
        full = att_call(eng, kernel, qkv)
        again = att_call(eng, kernel, qkv)
        assert full[0] == 0 and torch.equal(full[1], again[1]), (kernel, T)
        for b in (0, 3, 6):
            one = att_call(eng, kernel, qkv[b:b + 1].contiguous())
            assert one[0] == 0 and torch.equal(one[1], full[1][b:b + 1]), (kernel, T, b)


@pytest.mark.parametrize("T", [385, 641, 1600])
def test_mma16t_chunk_invariance(eng, T):
    """Each 64-key block is processed the same way whatever the chunk: the same bits for every chunk of 64 .. 384."""
    qkv = make_qkv(2, T, seed=T)
    rc, base, _, _, _ = att_call(eng, MMA16T, qkv)
    assert rc == 0
    for ch in range(64, 385, 64):
        rc, got, _, _, _ = att_call(eng, MMA16T, qkv, chunk=ch)
        assert rc == 0 and torch.equal(got, base), "chunk %d" % ch


def test_dispatch_boundary(eng):
    """The face forward runs the resident kernel up to 384 frames (12.8 s) and the tiled one from 385."""
    for T, k in ((384, MMA16P), (385, MMA16T)):
        qkv = make_qkv(1, T, seed=T)
        rc, auto, _, _, _ = att_call(eng, -1, qkv, fmt=2)
        rc2, forced, _, _, _ = att_call(eng, k, qkv, fmt=2)
        assert rc == 0 and rc2 == 0 and torch.equal(auto, forced), T


def test_truncation_bias(eng):
    """The tensor core's fp32 accumulator truncates toward zero.  On positive values (v ~ U[0.5, 1]) with flat-ish
    scores at T = 384 the mean signed error / |o| of both default kernels stays under BIAS_BAR, and the two agree."""
    qkv = make_qkv(4, 384, seed=91, shape="posv")
    ref = att_reference(qkv)["o"]
    means = []
    for k in (MMA16P, MMA16T):
        rc, o, _, _, _ = att_call(eng, k, qkv)
        assert rc == 0
        means.append(float(((o.double() - ref) / ref.abs()).mean()))
    print("att truncation bias T 384 positive v: mean err / |o| %.3g (mma16p), %.3g (mma16t)" % tuple(means))
    assert means[0] == means[1]
    assert abs(means[0]) <= BIAS_BAR, means


def test_attention_refused_without_launch(eng):
    """Requests a kernel cannot run come back as TS_ERR_INVALID before anything is launched or written."""
    cases = [
        (MMA16P, 385, 0, 0), (TF32, 385, 0, 0), (MMA16, 385, 0, 0), (FFMA, 3137, 0, 0),
        (5, 16, 0, 0), (-2, 16, 0, 0), (MMA16T, 16, 3, 0),
        (FFMA, 16, 2, 0), (TF32, 16, 2, 0), (MMA16, 16, 2, 0),
        (MMA16T, 16, 0, 32), (MMA16T, 16, 0, 448), (MMA16T, 16, 0, 100), (MMA16P, 16, 0, 64), (-1, 16, 0, 64),
    ]
    for kernel, T, fmt, chunk in cases:
        qkv = make_qkv(1, T, seed=1)
        out = torch.full((1, T, H * HD), SENT, device="cuda")
        hi = torch.full((1, T, H * HD), SENT, device="cuda")
        lo = hi.clone()
        rc, o, h, l, n = att_call(eng, kernel, qkv, fmt=fmt, chunk=chunk, out=out, hi=hi, lo=lo)
        assert rc == TS_ERR_INVALID and n == 0, (kernel, T, fmt, chunk, rc)
        assert (o == SENT).all() and (h == SENT).all() and (l == SENT).all()
    qkv = make_qkv(1, 16, seed=1)
    for B, T in ((0, 16), (1, 0)):
        a = DebugAtt(MMA16T, B, T, 0, 0)
        assert eng.L.ts_debug_attention(eng.h, C.byref(a), _lib.ptr(qkv), _lib.ptr(qkv), None, None, eng._s()) == TS_ERR_INVALID
    for fmt in (1, 2):                                              # missing planes
        a = DebugAtt(MMA16T, 1, 16, 0, fmt)
        assert eng.L.ts_debug_attention(eng.h, C.byref(a), _lib.ptr(qkv), _lib.ptr(qkv), None, None, eng._s()) == TS_ERR_INVALID
    a = DebugAtt(MMA16T, 1, 16, 0, 0)
    assert eng.L.ts_debug_attention(eng.h, C.byref(a), _lib.ptr(qkv), None, None, None, eng._s()) == TS_ERR_INVALID


# ---- positional conv ---------------------------------------------------------------------------------------------------
def split16_shift(mx):
    if mx == 0 or not math.isfinite(mx):
        return 0
    return min(100, max(-100, 14 - math.frexp(mx)[1]))


def make_pc(B, T, seed, w_max=None, x_range=None):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 768, generator=gen)
    if x_range is not None:
        lo, hi = x_range
        mag = torch.exp(torch.empty(B, T, 768).uniform_(math.log(lo), math.log(hi), generator=gen))
        x = torch.where(torch.rand(B, T, 768, generator=gen) < 0.5, -mag, mag)
    W = torch.randn(768, 48, 128, generator=gen) / math.sqrt(48 * 128)
    if w_max is not None:
        W = W / W.abs().max() * w_max if w_max else torch.zeros_like(W)
    bias = torch.randn(768, generator=gen) * 0.1
    return x.cuda(), W.contiguous(), bias


def pc_call(e, mode, x, W, bias, y=None, B=None, T=None):
    B, T = x.shape[0] if B is None else B, x.shape[1] if T is None else T
    y = torch.full((B, T, 768), float("nan"), device="cuda") if y is None else y
    Wn = W.numpy().astype(np.float32)
    bn = bias.numpy().astype(np.float32)
    n0 = e.launches
    rc = e.L.ts_debug_posconv(e.h, mode, _lib.ptr(x), Wn.ctypes.data_as(C.c_void_p), bn.ctypes.data_as(C.c_void_p),
                              _lib.ptr(y), B, T, e._s())
    torch.cuda.synchronize()
    return rc, y, e.launches - n0


def pc_reference(x, W, bias):
    """float64 per group: pre-activation z, y = GELU(z), S = sum|x||w|, sum|x| and sum|w| over every window."""
    B, T, _ = x.shape
    xp = torch.zeros(B, T + 128, 768, dtype=torch.float64, device="cuda")
    xp[:, 64:64 + T] = x.double()
    Wd = W.double().cuda()
    z, S, sx = (torch.empty(B, T, 768, dtype=torch.float64, device="cuda") for _ in range(3))
    for g in range(16):
        win = xp[:, :, 48 * g:48 * (g + 1)].unfold(1, 128, 1)[:, :T].reshape(B * T, 48 * 128)   # [B*T, c*128 + j]
        Wg = Wd[48 * g:48 * (g + 1)].reshape(48, 48 * 128)
        z[:, :, 48 * g:48 * (g + 1)] = (win @ Wg.T).view(B, T, 48)
        S[:, :, 48 * g:48 * (g + 1)] = (win.abs() @ Wg.abs().T).view(B, T, 48)
        sx[:, :, 48 * g:48 * (g + 1)] = win.abs().sum(1).view(B, T, 1)
    sw = Wd.abs().sum((1, 2)).view(1, 1, 768)
    b = bias.double().cuda().view(1, 1, 768)
    z = z + b
    y = 0.5 * z * (1 + torch.special.erf(z / math.sqrt(2)))
    return z, y, S, sx, sw, b.abs()


def pc_check(mode, x, W, bias, y, label, rms=True):
    assert torch.isfinite(y).all(), "%s: non-finite or unwritten outputs" % label
    z, yref, S, sx, sw, babs = pc_reference(x, W, bias)
    if mode == 0:
        rel = 6144 * 2.0 ** -24
        absu = 0.0
    else:
        rel = 3 * 2.0 ** -22 + 36 * 2.0 ** -22 + 32 * 2.0 ** -24
        absu = 2.0 ** -25 * (sw + sx / 2.0 ** split16_shift(float(W.abs().max())))
    tol = 1.13 * (rel * S + absu + 2.0 ** -22 * (S + babs)) + 2.0 ** -21 * z.abs()
    err = (y.double() - yref).abs()
    bad = err > tol
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        pytest.fail("%s: %d elements over the bar, first %s: got %.9g ref %.9g tol %.3g S %.3g" % (
            label, int(bad.sum()), i, float(y[i]), float(yref[i]), float(tol[i]), float(S[i])))
    pos = S > 0
    r = err[pos] / S[pos] if pos.any() else torch.zeros(1, dtype=torch.float64, device="cuda")
    st_rms, st_max = float(r.pow(2).mean().sqrt()), float(r.max())
    print("posconv %-20s mode %d B %2d T %4d: rms %.3g max %.3g (err / S), max err / bar %.3g" % (
        label, mode, x.shape[0], x.shape[1], st_rms, st_max, float((err / tol).max())))
    bar = RMS_BAR["pc"][0 if mode == 0 else 6]
    if rms:
        assert st_rms <= bar, "%s: RMS err / S %.3g over the bar %.3g" % (label, st_rms, bar)
    return st_rms, st_max


PC_LENGTHS = [1, 15, 16, 17, 63, 64, 65, 319, 320, 321, 640, 641, 3100]
PC_IDS = [(m, T, B) for m in (6, 0) for T in PC_LENGTHS for B in (1, 3)] + [(6, 300, 64), (0, 300, 64)]


@pytest.mark.parametrize("mode,T,B", PC_IDS, ids=["m%d-T%d-B%d" % p for p in PC_IDS])
def test_posconv_lengths(eng, mode, T, B):
    """Row blocks, the 320-row CTA boundary and its 127-row halo, and the production 64 clips x 10 s."""
    x, W, bias = make_pc(B, T, seed=zlib.crc32(b"pc%d" % T) + B)
    rc, y, n = pc_call(eng, mode, x, W, bias)
    assert rc == 0 and n == 3, eng.L.ts_last_error(eng.h)           # zeroing the pad rows, the staging fill, the conv
    pc_check(mode, x, W, bias, y, "lengths")


@pytest.mark.parametrize("mode", [6, 0])
@pytest.mark.parametrize("T,t0", [(65, 0), (65, 64), (321, 0), (321, 320)])
def test_posconv_impulse(eng, mode, T, t0):
    """One nonzero input (t0, channel 17 of group 5) = 1, zero bias: output (t, n) is GELU(W[n, 17, t0 - t + 64]) for
    the 48 channels of group 5 where that tap exists and exactly 0 everywhere else."""
    x = torch.zeros(1, T, 768, device="cuda")
    c = 5 * 48 + 17
    x[0, t0, c] = 1.0
    _, W, _ = make_pc(1, 1, seed=3)
    bias = torch.zeros(768)
    rc, y, _ = pc_call(eng, mode, x, W, bias)
    assert rc == 0
    want = torch.zeros(1, T, 768, dtype=torch.float64)
    t = torch.arange(T)
    j = t0 - t + 64
    ok = (j >= 0) & (j < 128)
    w = W[5 * 48:6 * 48, 17, :].double()                               # [48, 128]
    zz = w[:, j[ok]].T                                                 # [rows, 48]
    want[0, t[ok], 5 * 48:6 * 48] = 0.5 * zz * (1 + torch.special.erf(zz / math.sqrt(2)))
    got = y.cpu().double()
    assert torch.equal(got == 0, want == 0), "impulse at %d: nonzero pattern" % t0
    assert ((got - want).abs() <= 2.0 ** -20 * want.abs()).all(), "impulse at %d: values" % t0


@pytest.mark.parametrize("mode", [6, 0])
@pytest.mark.parametrize("wmax", ["2^-20", "2^-30", "7e4", "0"])
def test_posconv_weight_scale(eng, mode, wmax):
    """Tiny, huge and all-zero layers: the pre-split weights are scaled by a power of two that puts max|W| in
    [2^13, 2^14), so they meet the same bars (an all-zero layer gives GELU(bias))."""
    w = {"2^-20": 2.0 ** -20, "2^-30": 2.0 ** -30, "7e4": 7e4, "0": 0.0}[wmax]
    x, W, bias = make_pc(2, 200, seed=31, w_max=w)
    bias = bias * (w if w else 1.0)
    rc, y, _ = pc_call(eng, mode, x, W, bias)
    assert rc == 0
    pc_check(mode, x, W, bias, y, "w_" + wmax)


@pytest.mark.parametrize("mode", [6, 0])
@pytest.mark.parametrize("mag", ["6e4", "1e-6"])
def test_posconv_input_magnitude(eng, mode, mag):
    """|x| up to 6e4 (inside the fp16 range) and down to 1e-6 (the split's absolute underflow term)."""
    rng = {"6e4": (1e2, 6e4), "1e-6": (1e-7, 1e-6)}[mag]
    x, W, bias = make_pc(2, 200, seed=21, x_range=rng)
    bias = bias * rng[1] * 0.1
    rc, y, _ = pc_call(eng, mode, x, W, bias)
    assert rc == 0
    pc_check(mode, x, W, bias, y, "x_" + mag, rms=not (mode == 6 and mag == "1e-6"))


def test_posconv_exact(eng):
    """Same bits on a second call, for an item alone as inside a batch of 7, and in modes 1 and 6 (one kernel)."""
    x, W, bias = make_pc(7, 333, seed=41)
    for mode in (6, 0):
        full = pc_call(eng, mode, x, W, bias)[1]
        assert torch.equal(full, pc_call(eng, mode, x, W, bias)[1]), mode
        for b in (0, 3, 6):
            one = pc_call(eng, mode, x[b:b + 1].contiguous(), W, bias)[1]
            assert torch.equal(one, full[b:b + 1]), (mode, b)
        if mode == 6:
            assert torch.equal(pc_call(eng, 1, x, W, bias)[1], full)


def test_posconv_refused_without_launch(eng):
    x, W, bias = make_pc(1, 16, seed=1)
    y = torch.full((1, 16, 768), SENT, device="cuda")
    for mode, B, T in ((2, 1, 16), (3, 1, 16), (7, 1, 16), (-1, 1, 16), (6, 0, 16), (6, 1, 0)):
        rc, out, n = pc_call(eng, mode, x, W, bias, y=y, B=B, T=T)
        assert rc == TS_ERR_INVALID and n == 0 and (out == SENT).all(), (mode, B, T)
    a = eng.L.ts_debug_posconv(eng.h, 6, _lib.ptr(x), None, None, _lib.ptr(y), 1, 16, eng._s())
    assert a == TS_ERR_INVALID
