"""GPU (-m gpu): the dense conv kernels on their own -- the wgmma kernel (csrc/gemm_tc.cu) on fp16-split (mode 6) and
3xTF32 (mode 1) operands and the FFMA kernel (csrc/gemm.cu, mode 0) -- through ts_debug_conv1d, which builds one Conv1d
layer the way the nets build it (activation layouts, operand splits, per-layer weight scale) and calls the chosen kernel
directly.  Every result is compared with torch's conv1d restated in float64 on the same fp32 inputs, followed by bias,
residual and the activation.

Accuracy bar, per element (derivation; S = sum_k |x_k||w_k| over the window, all terms relative to S unless noted):
  * operands: the fp16 split keeps 11 + 11 significant bits round-to-nearest, so each of x and w is represented to
    2^-22 while its low plane is normal, and the dropped lo*lo product is below 2^-22: 3 * 2^-22 per product.  The 3xTF32
    split truncates lo to tf32 (2^-20 of hi) and drops lo*lo: 3 * 2^-20.  The FFMA kernel uses the fp32 values.
  * tensor-core accumulation: each wgmma (3 per k-step, 4 k-steps per 128-byte k-block) adds into the fp32 accumulator
    with truncation, at most 2^-22 of the chunk's partial S each: 12 * cb * 2^-22 for cb k-blocks per chunk (K = 256:
    cb = 4 fp16 / 8 tf32 k-blocks).  The K / 256 chunks are then added round-to-nearest: nchunks * 2^-24.
    FFMA: a chain of K fp32 FMAs, gamma_K = K * 2^-24.
  * underflow (fp16 split, absolute): a low plane that is subnormal leaves an absolute error of 2^-25 per operand, i.e.
    2^-25 * sum|w| for the activation and 2^-25 / 2^shift * sum|x| for the weights scaled by 2^shift (split16_shift).
  * epilogue: the unscale, bias and residual adds round at 2^-24 each: 2^-22 * (S + |bias| + |res|) absolute.
  * activation: |f'| <= 1.13 (GELU) multiplies the above; its own fp32 evaluation adds 2^-21 * |pre-activation|.
  * an output read back from fp16 planes adds its representation error, 2^-22 |y| + 2^-25.
A dropped hi*lo product (2^-12 of each product), a wrong tap, row or swizzle, or a lost partial chunk each move the
error by orders of magnitude over the statistical bar below (and the latter three over the per-element bar).

Statistical bar: the RMS over the outputs of |error| / S is pinned per mode at 4x the largest value measured over the
cases below on one H100 80GB HBM3 (700 W power limit): 9.3e-8 in mode 6, 2.2e-7 in mode 1, 3.1e-8 in mode 0 (the
smallest K give the largest values).  A dropped hi*lo product alone would give about 2^-12 / sqrt(K), 4.4e-6 at
K = 3072, twelve times the mode-6 bar.  Cases whose error is dominated by the absolute underflow term (fp16 activations
of 1e-6 and below: RMS 1e-3 and 3e-2 measured) are checked against the per-element bar only.  Every case prints its
statistics ("dense ..." lines, pytest -s).

Also checked: pad rows of the output stay zero and rows / columns the layer does not own keep a sentinel (the other phase
of a transposed conv, columns outside [coff, coff + N)); outputs are finite although the input's tail rows are NaN; the
output's split planes (mode 6: h = fp16(y), l = fp16(y - h) bit for bit; mode 1: hi has its 13 low bits clear); two
calls give the same bits and an item gives the same bits alone as inside a batch of 7; the round-to-nearest chunking
measurably reduces the tensor core's truncation bias; layers with max|W| of 2^-20, 2^-30 and 7e4 meet the same bars;
invalid geometries return TS_ERR_INVALID without a launch."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

from talkshow_b200 import _lib

pytestmark = pytest.mark.gpu

TS_ERR_INVALID = 1
NONE, RELU, LRELU, GELU = 0, 1, 2, 3
SENT = 1234.5                 # fp32 sentinel of the rows / columns a layer must not write
SENT16 = 0x5A5A               # fp16-plane sentinel (bits)
# RMS of |error| / S, 4x the largest value measured on one H100 80GB HBM3 (700 W); see the module docstring
RMS_BAR = {6: 4 * 9.3e-8, 1: 4 * 2.2e-7, 0: 4 * 3.1e-8}
# mean signed error / S of a K = 3072 fp16-split layer on positive operands: -1.73e-6 measured (H100 80GB HBM3, 700 W)
CHUNK_MEAN_BAR = 2 * 1.73e-6
_FIELDS = ("mode", "B", "T", "C", "x_pad", "x_tail", "N", "k", "stride", "pd", "T_out", "act", "y_T", "y_C", "y_pad",
           "y_tmul", "y_toff", "coff", "y_split", "res_pad", "res_split", "chunk", "planes_only")


class DebugConv(C.Structure):
    _fields_ = [(f, C.c_int32) for f in _FIELDS]


def pad4(n):
    return (n + 3) & ~3


def geo(C, N, k=1, stride=1, pd=0, B=2, T=100, x_pad=None, x_tail=0, T_out=None, act=NONE, y_T=None, y_C=None, y_pad=0,
        y_tmul=1, y_toff=0, coff=0, y_split=0, res=False, res_pad=0, res_split=0, planes_only=0):
    g = dict(C=C, N=N, k=k, stride=stride, pd=pd, B=B, T=T, x_pad=pd if x_pad is None else x_pad, x_tail=x_tail, act=act,
             y_pad=y_pad, y_tmul=y_tmul, y_toff=y_toff, coff=coff, y_split=y_split, res=res, res_pad=res_pad,
             res_split=res_split, planes_only=planes_only)
    g["T_out"] = (T + 2 * pd - k) // stride + 1 if T_out is None else T_out
    g["y_T"] = (g["T_out"] - 1) * y_tmul + y_toff + 1 if y_T is None else y_T
    g["y_C"] = coff + pad4(N) if y_C is None else y_C
    return g


def split16_shift(mx):
    """The weight scale exponent the fp16 split should use: max|W| * 2^shift in [2^13, 2^14)."""
    if mx == 0 or not math.isfinite(mx):
        return 0
    return min(100, max(-100, 14 - math.frexp(mx)[1]))


@pytest.fixture(scope="module")
def eng():
    from talkshow_b200.engine import Engine

    torch.set_grad_enabled(False)
    e = Engine(0)
    yield e
    torch.cuda.synchronize()
    e.close()


def make_inputs(g, seed, x_scale=1.0, w_max=None, x_range=None, positive=False, device="cuda"):
    gen = torch.Generator().manual_seed(seed)
    B, T, Cc, N, k = g["B"], g["T"], g["C"], g["N"], g["k"]
    if positive:
        x = torch.rand(B, T, Cc, generator=gen)
        W = torch.rand(N, Cc, k, generator=gen) / (Cc * k)
    else:
        x = torch.randn(B, T, Cc, generator=gen) * x_scale
        W = torch.randn(N, Cc, k, generator=gen) / math.sqrt(Cc * k)
    if x_range is not None:                     # magnitudes log-uniform in [lo, hi], random signs
        lo, hi = x_range
        mag = torch.exp(torch.empty(B, T, Cc).uniform_(math.log(lo), math.log(hi), generator=gen))
        x = torch.where(torch.rand(B, T, Cc, generator=gen) < 0.5, -mag, mag)
    if w_max is not None:
        W = W / W.abs().max() * w_max if w_max else torch.zeros_like(W)
    bias = torch.randn(N, generator=gen) * 0.1
    res = torch.randn(B, g["T_out"], N, generator=gen) * 0.5 if g["res"] else None
    return x.to(device), W.contiguous(), bias, None if res is None else res.to(device)


def _buffers(g, mode):
    """Output buffers as the caller hands them in: pad rows zero, every other element a sentinel."""
    B, rows, yC, yp = g["B"], g["y_T"] + 2 * g["y_pad"], g["y_C"], g["y_pad"]
    y = torch.full((B, rows, yC), SENT, device="cuda")
    y[:, :yp] = 0
    y[:, rows - yp:] = 0
    if mode == 6:
        hi = torch.full((B, rows, yC), SENT16, dtype=torch.int16, device="cuda")
        lo = hi.clone()
    else:
        hi, lo = y.clone(), y.clone()
    for p in (hi, lo):
        p[:, :yp] = 0
        p[:, rows - yp:] = 0
    return y, hi, lo


def call(e, mode, g, x, W, bias, res, chunk=0, bufs=None, planes_only=None):
    """-> (status, y, plane_hi, plane_lo, launches issued)."""
    y, hi, lo = _buffers(g, mode) if bufs is None else bufs
    a = DebugConv(**{f: 0 for f in _FIELDS})
    for f in _FIELDS:
        if f in g:
            setattr(a, f, int(g[f]))
    a.mode, a.chunk = mode, chunk
    a.planes_only = (g["planes_only"] if mode == 6 else 0) if planes_only is None else planes_only
    a.res_pad, a.res_split = g["res_pad"], g["res_split"]
    Wn = W.numpy().astype(np.float32)
    bn = None if bias is None else bias.numpy().astype(np.float32)
    n0 = e.launches
    rc = e.L.ts_debug_conv1d(e.h, C.byref(a), _lib.ptr(x), Wn.ctypes.data_as(C.c_void_p),
                             None if bn is None else bn.ctypes.data_as(C.c_void_p), _lib.ptr(res), _lib.ptr(y),
                             _lib.ptr(hi), _lib.ptr(lo), e._s())
    torch.cuda.synchronize()
    return rc, y, hi, lo, e.launches - n0


def reference(g, x, W, bias, res):
    """float64 on the GPU: pre-activation z, activation y, S = sum|x||w|, sum|x| and sum|w| over every window."""
    B, T, Cc = x.shape
    k, s, pd, To = g["k"], g["stride"], g["pd"], g["T_out"]
    right = max(0, (To - 1) * s + k - pd - T)
    xp = torch.zeros(B, pd + T + right, Cc, dtype=torch.float64, device=x.device)
    xp[:, pd:pd + T] = x.double()
    win = xp.unfold(1, k, s)[:, :To].reshape(B * To, Cc * k)          # [B*To, C*k], c-major like W.reshape
    Wd = W.double().to(x.device).reshape(W.shape[0], Cc * k)
    z = (win @ Wd.T).view(B, To, -1)
    S = (win.abs() @ Wd.abs().T).view(B, To, -1)
    sx = win.abs().sum(1).view(B, To, 1)
    sw = Wd.abs().sum(1).view(1, 1, -1)
    extra = torch.zeros_like(z)
    if bias is not None:
        b = bias.double().to(x.device).view(1, 1, -1)
        z, extra = z + b, extra + b.abs()
    if res is not None:
        z, extra = z + res.double(), extra + res.double().abs()
    act = g["act"]
    if act == RELU:
        y = z.clamp_min(0)
    elif act == LRELU:
        y = torch.where(z > 0, z, 0.2 * z)
    elif act == GELU:
        y = 0.5 * z * (1 + torch.special.erf(z / math.sqrt(2)))
    else:
        y = z
    return z, y, S, sx, sw, extra


def bound(mode, K, chunk=0):
    if mode == 0:
        return K * 2.0 ** -24
    bk = 64 if mode == 6 else 32
    nk = K // bk
    cb = min(nk, chunk or 256 // bk)
    nch = -(-nk // cb)
    prod = 3 * 2.0 ** -22 if mode == 6 else 3 * 2.0 ** -20
    return prod + 12 * cb * 2.0 ** -22 + nch * 2.0 ** -24


def written_mask(g, shape):
    m = torch.zeros(shape, dtype=torch.bool, device="cuda")
    rows = torch.arange(g["T_out"], device="cuda") * g["y_tmul"] + g["y_toff"] + g["y_pad"]
    m[:, rows, g["coff"]:g["coff"] + g["N"]] = True
    return m, rows


def select(buf, g, rows):
    return buf[:, rows, g["coff"]:g["coff"] + g["N"]]


def check(mode, g, x, W, bias, res, out, chunk=0, label="", rms=True, init=None):
    """Accuracy, placement and planes of one call's result; returns (rms, max) of |error| / S."""
    rc, y, hi, lo, _ = out
    assert rc == 0, label
    z, yref, S, sx, sw, extra = reference(g, x, W, bias, res)
    K = g["C"] * g["k"]
    planes_out = g["y_split"] and mode == 6 and (g["planes_only"] & 2)
    y_full = not g["y_split"] or (mode == 6 and not planes_out)
    mask, rows = written_mask(g, y.shape)
    init = init or _buffers(g, mode)
    # placement: every element outside the layer's rows / columns keeps what the caller put there (zero pad rows included)
    for name, buf, ini, written in (("y", y, init[0], y_full), ("hi", hi, init[1], bool(g["y_split"])),
                                    ("lo", lo, init[2], bool(g["y_split"]))):
        keep = ~mask if written else torch.ones_like(mask)
        assert torch.equal(buf[keep], ini[keep]), "%s: %s written outside its rows / columns" % (label, name)
    rep = torch.zeros_like(yref)
    if y_full:
        got = select(y, g, rows).double()
    elif mode == 6:
        got = (select(hi, g, rows).view(torch.float16).double() + select(lo, g, rows).view(torch.float16).double())
        rep = 2.0 ** -22 * yref.abs() + 2.0 ** -25
    else:
        h, l = select(hi, g, rows), select(lo, g, rows)
        assert (h.view(torch.int32) & 0x1FFF).eq(0).all(), "%s: 3xTF32 hi plane with low mantissa bits set" % label
        got = h.double() + l.double()
    if g["y_split"] and mode == 6 and y_full:        # fp16 planes of the returned value, bit for bit
        yn = select(y, g, rows).cpu().numpy()
        h16 = yn.astype(np.float16)
        l16 = (yn - h16.astype(np.float32)).astype(np.float16)
        assert np.array_equal(select(hi, g, rows).cpu().numpy().view(np.uint16), h16.view(np.uint16)), label
        assert np.array_equal(select(lo, g, rows).cpu().numpy().view(np.uint16), l16.view(np.uint16)), label
    assert torch.isfinite(got).all(), "%s: non-finite outputs" % label
    absu = 0.0
    if mode == 6:
        sc = 2.0 ** split16_shift(float(W.abs().max()))
        absu = 2.0 ** -25 * (sw + sx / sc)
    tol = 1.13 * (bound(mode, K, chunk) * S + absu + 2.0 ** -22 * (S + extra)) + 2.0 ** -21 * z.abs() + rep
    err = (got - yref).abs()
    bad = err > tol
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail("%s: %d elements over the bar, first %s: got %.9g ref %.9g tol %.3g S %.3g" % (
            label, int(bad.sum()), i, float(got[tuple(i)]), float(yref[tuple(i)]), float(tol[tuple(i)]), float(S[tuple(i)])))
    pos = S > 0
    r = (err[pos] / S[pos]) if pos.any() else torch.zeros(1, dtype=torch.float64, device="cuda")
    st_rms, st_max = float(r.pow(2).mean().sqrt()), float(r.max())
    print("dense %-28s mode %d K %5d N %4d rows %7d: rms %.3g max %.3g (err / S)" % (label, mode, K, g["N"],
                                                                                        g["B"] * g["T_out"], st_rms, st_max))
    if rms:
        assert st_rms <= RMS_BAR[mode], "%s: RMS err / S %.3g over the bar %.3g" % (label, st_rms, RMS_BAR[mode])
    return st_rms, st_max


# ---- production geometries (face.cu face_run, convstack.cu run_stack / run_up / run_decoder, pixelcnn_tf.cu tf_forward) --
D = 256   # body prior width
PROD = {
    # wav2vec2 feature extractor: odd T, one tail row so rows per item are even; fp16 planes only in and out; GELU
    "w2v_k3s2": (geo(512, 512, k=3, stride=2, T=399, x_tail=1, act=GELU, y_split=1, planes_only=3), (6, 1, 0)),
    "w2v_k2s2": (geo(512, 512, k=2, stride=2, B=3, T=49, x_tail=1, act=GELU, y_split=1, planes_only=3), (6, 1, 0)),
    # transformer linears (frame rows)
    "fproj_ypad64": (geo(512, 768, T=150, y_pad=64), (6, 1, 0)),
    "qkv": (geo(768, 2304, T=120), (6, 1, 0)),
    "out_res": (geo(768, 768, T=120, res=True, res_split=1), (6, 1, 0)),
    "ff1_gelu": (geo(768, 3072, T=120, act=GELU, y_split=1), (6, 1, 0)),
    "ff2_res": (geo(3072, 768, T=120, res=True, res_split=1), (6, 1, 0)),
    "feat_map_320": (geo(768, 256, T=120, y_C=320, y_pad=1, y_split=1), (6, 1, 0)),
    # first_net / decoder convs
    "first_net_c320": (geo(320, 256, k=3, pd=1, T=120), (6, 1, 0)),
    "first_net_c256": (geo(256, 256, k=3, pd=1, T=120), (6, 1, 0)),
    "decoder_n64": (geo(256, 64, k=3, pd=1, T=120), (6, 1, 0)),
    # VQ decoder
    "aft_vq_k64": (geo(64, 1024, T=22, y_pad=1, y_split=1), (6, 1, 0)),
    "res_stack_1024": (geo(1024, 1024, k=3, pd=1, T=22, y_pad=1, y_split=1, act=LRELU), (6, 1, 0)),
    "res_stack_fin_256": (geo(256, 256, k=3, pd=1, T=88, y_pad=1, y_split=1, act=RELU, res=True, res_pad=1, res_split=1),
                          (6, 1, 0)),
    "project_n39": (geo(256, 39, T=88, y_C=40), (6, 1, 0)),
    "project_n90": (geo(256, 90, T=88, y_C=92), (6, 1, 0)),
    # teacher-forced prior over cells (R = 2T rows per item, TF_PAD = 6 zero cells in front of every sample)
    "tf_vert_l0": (geo(D, 4 * D, k=6, stride=2, pd=6, x_pad=6, T=2 * 44, T_out=44, y_split=1), (6, 1, 0)),
    "tf_vert": (geo(D, 4 * D, k=4, stride=2, pd=2, x_pad=6, T=2 * 44, T_out=44, y_split=1), (6, 1, 0)),
    "tf_horiz_l0": (geo(D, 4 * D, k=1, stride=2, pd=0, x_pad=6, T=2 * 44, T_out=44), (6, 1, 0)),
    "tf_horiz": (geo(D, 4 * D, k=2, stride=2, pd=0, x_pad=6, T=2 * 44, T_out=44), (6, 1, 0)),
    "tf_v2h_res": (geo(2 * D, 2 * D, T=2 * 44, res=True), (6, 1, 0)),
}
PROD_IDS = [(n, m) for n, (_, modes) in PROD.items() for m in modes]


@pytest.mark.parametrize("name,mode", PROD_IDS, ids=["%s-m%d" % p for p in PROD_IDS])
def test_production_geometry(eng, name, mode):
    g = PROD[name][0]
    x, W, bias, res = make_inputs(g, seed=zlib.crc32(name.encode()))
    out = call(eng, mode, g, x, W, bias, res)
    check(mode, g, x, W, bias, res, out, label=name)
    again = call(eng, mode, g, x, W, bias, res)                     # determinism: the same bits every call
    for a, b in zip(out[1:4], again[1:4]):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("mode", [6, 1, 0])
def test_transposed_conv_phases_share_one_buffer(eng, mode):
    """ConvTranspose1d(k 4, s 2, p 1) as run_up runs it: the even phase (k 2, pd 1) writes rows 2m, the odd phase
    (k 2, pd 0) rows 2m + 1 of the same buffer; each leaves the other's rows alone."""
    T = 44
    ev = geo(512, 256, k=2, pd=1, x_pad=1, T=T, T_out=T, y_T=2 * T, y_pad=1, y_tmul=2, y_toff=0, y_split=1, act=LRELU)
    od = dict(ev, pd=0, y_toff=1)
    x, We, bias, _ = make_inputs(ev, seed=11)
    _, Wo, bias_o, _ = make_inputs(ev, seed=12)
    bufs = _buffers(ev, mode)
    init = tuple(b.clone() for b in bufs)
    out = call(eng, mode, ev, x, We, bias, None, bufs=bufs)
    check(mode, ev, x, We, bias, None, out, label="up_even", init=init)
    mid = tuple(b.clone() for b in bufs)
    out = call(eng, mode, od, x, Wo, bias_o, None, bufs=bufs)
    check(mode, od, x, Wo, bias_o, None, out, label="up_odd", init=mid)
    me, _ = written_mask(ev, bufs[0].shape)
    for b, m0 in zip(bufs, mid):                                    # the odd call left the even rows alone
        assert torch.equal(b[me], m0[me])


# ---- edges ------------------------------------------------------------------------------------------------------------
EDGES = {
    "rows1": (geo(256, 128, B=1, T=1), (6, 1, 0)),
    "rows127": (geo(256, 128, B=1, T=127), (6, 1, 0)),
    "rows128": (geo(256, 128, B=1, T=128), (6, 1, 0)),
    "rows129": (geo(256, 128, B=1, T=129), (6, 1, 0)),
    "b7_t37_k3": (geo(256, 128, k=3, pd=1, B=7, T=37), (6, 1, 0)),
    "K64": (geo(64, 128), (6, 1, 0)),
    "K192": (geo(192, 128), (6, 1, 0)),
    "K256": (geo(256, 128), (6, 1, 0)),
    "K320": (geo(320, 128), (6, 1, 0)),
    "K1536": (geo(512, 128, k=3, pd=1), (6, 1, 0)),
    "K3072": (geo(3072, 128), (6, 1, 0)),
    "K32": (geo(32, 128), (1, 0)),
    "K96": (geo(96, 128), (1, 0)),
    "N1": (geo(256, 1), (6, 1, 0)),
    "N3": (geo(256, 3), (6, 1, 0)),
    "N4": (geo(256, 4), (6, 1, 0)),
    "N127": (geo(256, 127), (6, 1, 0)),
    "N128": (geo(256, 128), (6, 1, 0)),
    "N129": (geo(256, 129, y_split=1), (6, 1, 0)),
    "N260": (geo(256, 260, y_split=1), (6, 1, 0)),
    "Tout1": (geo(256, 64, k=3, stride=2, B=3, T=4, T_out=1, x_tail=0), (6, 1, 0)),
    "coff68": (geo(256, 64, k=3, pd=1, coff=68, y_C=200, y_split=1), (6, 1, 0)),
    "act_none": (geo(256, 64, k=3, pd=1, act=NONE), (6, 1, 0)),
    "act_relu": (geo(256, 64, k=3, pd=1, act=RELU, res=True, res_pad=1), (6, 1, 0)),
    "act_lrelu": (geo(256, 64, k=3, pd=1, act=LRELU, res=True), (6, 1, 0)),
    "act_gelu": (geo(256, 64, k=3, pd=1, act=GELU, y_split=1), (6, 1, 0)),
}
EDGE_IDS = [(n, m) for n, (_, modes) in EDGES.items() for m in modes]


@pytest.mark.parametrize("name,mode", EDGE_IDS, ids=["%s-m%d" % p for p in EDGE_IDS])
def test_edge_geometry(eng, name, mode):
    g = EDGES[name][0]
    x, W, bias, res = make_inputs(g, seed=zlib.crc32(name.encode()) + 1)
    check(mode, g, x, W, bias, res, call(eng, mode, g, x, W, bias, res), label=name)


@pytest.mark.parametrize("mode", [6, 1])
def test_large_m(eng, mode):
    """More than 10^6 GEMM rows (8200 row tiles): every tile lands where it belongs."""
    g = geo(64, 4, B=3, T=350_001, x_tail=1, res=True)
    assert g["B"] * (g["T"] + 1) > 10 ** 6
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(g["B"], g["T"], 64, device="cuda", generator=gen)
    W = torch.randn(4, 64, 1) / 8
    bias = torch.randn(4) * 0.1
    res = torch.randn(g["B"], g["T_out"], 4, device="cuda", generator=gen)
    check(mode, g, x, W, bias, res, call(eng, mode, g, x, W, bias, res), label="large_m")


@pytest.mark.parametrize("mode", [6, 1, 0])
@pytest.mark.parametrize("mag", ["6e4", "1e-6", "1e-9"])
def test_input_magnitude(eng, mode, mag):
    """|x| up to 6e4 (inside the fp16 range) and down to 1e-9 (fp16 planes underflow: the absolute term of the bar)."""
    g = geo(512, 128, k=3, pd=1, act=LRELU)
    rng = {"6e4": (1e2, 6e4), "1e-6": (1e-7, 1e-6), "1e-9": (1e-10, 1e-9)}[mag]
    x, W, bias, res = make_inputs(g, seed=21, x_range=rng)
    bias = bias * rng[1] * 0.1
    check(mode, g, x, W, bias, res, call(eng, mode, g, x, W, bias, res), label="x_" + mag, rms=not (mode == 6 and mag != "6e4"))


@pytest.mark.parametrize("mode", [6, 1, 0])
@pytest.mark.parametrize("wmax", ["2^-20", "2^-30", "7e4", "0"])
def test_weight_scale(eng, mode, wmax):
    """The fp16 split scales every layer by a power of two that puts max|W| in [2^13, 2^14): tiny and huge layers meet
    the same relative bars as an ordinary one (no subnormal low plane, no fp16 overflow), an all-zero layer gives
    act(bias + res).  A layer scaled by 2^-20 or 2^-30 (weights, bias and residual) gives exactly the outputs of the
    layer with max|W| = 1 times that power of two, bit for bit: the scale only moves exponents."""
    w = {"2^-20": 2.0 ** -20, "2^-30": 2.0 ** -30, "7e4": 7e4, "0": 0.0}[wmax]
    g = geo(768, 256, k=1, T=120, res=True, y_split=int(w < 1))      # fp16 output planes hold |y| < 65504 only
    x, W, bias, res = make_inputs(g, seed=31, w_max=w)
    scale = w if w else 1.0
    bias, res = bias * scale, res * scale
    check(mode, g, x, W, bias, res, call(eng, mode, g, x, W, bias, res), label="w_" + wmax)
    if w in (2.0 ** -20, 2.0 ** -30):
        g0 = dict(g, y_split=0)
        _, W1, b1, r1 = make_inputs(g0, seed=31, w_max=1.0)
        assert float(W1.abs().max()) == 1.0 and torch.equal(W1 * w, W)
        _, rows = written_mask(g0, (g0["B"], g0["y_T"], g0["y_C"]))
        unit = select(call(eng, mode, g0, x, W1, b1, r1)[1], g0, rows)
        scaled = select(call(eng, mode, g0, x, W1 * w, b1 * w, r1 * w)[1], g0, rows)
        assert torch.equal(scaled, unit * w), "w_%s: not the unit layer's outputs scaled" % wmax


def test_position_independence(eng):
    """An item gives the same bits alone (B = 1) as inside a batch of 7 whose items straddle the 128-row tiles."""
    for mode in (6, 1, 0):
        g7 = geo(256, 128, k=3, pd=1, B=7, T=37, y_pad=1, y_split=1, act=GELU)
        x, W, bias, _ = make_inputs(g7, seed=41)
        full = call(eng, mode, g7, x, W, bias, None)
        assert full[0] == 0
        for b in (0, 3, 6):
            g1 = dict(g7, B=1)
            one = call(eng, mode, g1, x[b:b + 1].contiguous(), W, bias, None)
            assert one[0] == 0
            for a, c in zip(full[1:4], one[1:4]):
                assert torch.equal(a[b:b + 1], c), (mode, b)


def test_chunking(eng):
    """The wgmma accumulator truncates toward zero, so the kernel adds chunks of K = 256 round-to-nearest.  With positive
    operands at K = 3072 (fp16 split) the mean signed error / S stays under CHUNK_MEAN_BAR, and one chunk over the whole K
    (chunk = 48 k-blocks) is at least 3x worse.  Measured on one H100 80GB HBM3 (700 W): -1.73e-6 with K = 256 chunks,
    -2.31e-5 with one chunk."""
    g = geo(3072, 256, T=256)
    x, W, bias, _ = make_inputs(g, seed=51, positive=True)
    z, _, S, _, _, _ = reference(g, x, W, None, None)
    means = []
    for chunk in (0, 48):
        rc, y, _, _, _ = call(eng, 6, g, x, W, None, None, chunk=chunk)
        assert rc == 0
        means.append(float(((y.double() - z) / S).mean()))
    print("dense chunking K 3072 positive: mean err / S %.3g (K 256 chunks), %.3g (one chunk)" % tuple(means))
    assert abs(means[0]) <= CHUNK_MEAN_BAR, means
    assert abs(means[1]) >= 3 * abs(means[0]), means


def test_invalid_geometry_refused_without_launch(eng):
    """Geometries a kernel cannot run come back as TS_ERR_INVALID before anything is launched or written."""
    base = geo(256, 64)
    x, W, bias, _ = make_inputs(base, seed=61)
    cases = [
        (6, dict(y_C=66), "y_C"), (1, dict(y_C=66), "y_C"),
        (6, dict(coff=2, y_C=68), "coff"), (1, dict(coff=2, y_C=68), "coff"),
        (6, dict(C=96), "k-block"), (1, dict(C=80), "k-block"),
        (6, dict(k=2, stride=2, T=99, T_out=49), "stride"), (1, dict(k=3, stride=2, x_pad=1, pd=0, T=100, T_out=49), "stride"),
        (3, {}, "mode"), (2, {}, "mode"), (7, {}, "mode"), (-1, {}, "mode"),
        (0, dict(C=254), "C % 4"),
        (6, dict(T_out=101), "window"),
    ]
    for mode, kw, why in cases:
        g = dict(base, **kw)
        xx = torch.randn(g["B"], g["T"], g["C"], device="cuda")
        WW = torch.randn(g["N"], g["C"], g["k"]) / 16
        bufs = _buffers(g, mode if mode in (0, 1, 6) else 6)
        init = tuple(b.clone() for b in bufs)
        rc, y, hi, lo, launched = call(eng, mode, g, xx, WW, bias, None, bufs=bufs)
        assert rc == TS_ERR_INVALID, (mode, kw, rc)
        assert launched == 0, (mode, kw)
        assert all(torch.equal(a, b) for a, b in zip((y, hi, lo), init)), (mode, kw)
        assert why.split()[0].lower() in eng.L.ts_last_error(eng.h).decode().lower() or why in ("window",), (
            why, eng.L.ts_last_error(eng.h))
    bufs = _buffers(base, 1)
    assert call(eng, 1, base, x, W, bias, None, bufs=bufs, planes_only=1)[0] == TS_ERR_INVALID
    assert "planes" in eng.L.ts_last_error(eng.h).decode()
    # the engine's kernel setting is untouched by the debug calls
    g = geo(256, 64, k=3, pd=1)
    assert call(eng, 6, g, x, W, bias, None)[0] == 0
    assert eng.L.ts_set_tensor_cores(eng.h, 6) == 0
