"""GPU (-m gpu): the face regressor's small front-end kernels and the VQ code argmin on their own -- conv0 + GroupNorm +
GELU (conv0_stats_kernel + conv0_apply_kernel, csrc/face.cu) through ts_debug_conv0_gn, the 50 -> 30 fps interpolation
(interp_kernel) through ts_debug_interp, every LayerNorm of the face net (ln_pre_kernel) through ts_debug_layernorm, and
vq_argmin_kernel (csrc/gemm.cu) through ts_debug_vq_argmin.  Each entry stages the data as the production path does and
runs the production launches.  Every result is compared with a float64 evaluation of the same fp32 inputs.
u = 2^-24 (fp32 unit roundoff) below.

conv0 + GroupNorm + GELU bar, per element (y_t = sum_j w_j x_{5t+j} exactly, S_t = sum_j |w_j| |x_{5t+j}|, mean / var /
rstd = 1 / sqrt(var + 1e-5) of the exact y over the clip, a_t = |y_t - mean| rstd the normalised magnitude):
  * the 10-tap fp32 FMA chain: |dy_t| <= D_t = 10 u S_t;
  * the statistics (fp64 sums of the kernel's y, fp64 rounding negligible): |dmean| <= Dm = mean_t D_t; the variance
    moves by at most 2 sd max_t D_t + (max_t D_t)^2 (the deviations' sum is zero, so the mean's error enters squared)
    plus the fp64 cancellation of E[y^2] - mean^2, 4 * 2^-53 E[y^2]; the relative error of rstd is half the variance's
    over (var + eps) plus its fp32 rounding, u;
  * mu is rounded to fp32: 2^-24 |mean| rstd |g| (the dominant term for a DC-heavy clip; the reference's fp32 GroupNorm
    has it too);
  * (y - mu) rstd g + b in fp32: |g| rstd (D_t + Dm + 2 u |mean|) + |g| a_t (e_rstd + 4 u) + u (|b| + |z|);
  * GELU: slope <= 1.13 times all of the above, plus its own fp32 evaluation (erff 2 ulp, the argument and the products
    rounded): 2^-21 |z| + 2^-22 |GELU(z)|;
  * the split formats: mode 1 stores hi + lo = v exactly; mode 6 stores h + l with 22 significant bits while l is
    normal and an absolute 2^-25 below: + 2^-22 |v| + 2^-25.
Exact: a silent clip and a constant (DC) wave give GELU(beta) at every t (the variance clamps to 0, y - mu = 0); samples
past the last window are never read (perturbing them gives the same bits); the tail row of an odd T0 stays NaN in every
plane; repeated calls, an item alone vs inside a batch, and the three output formats of one input agree bit for bit
where each clip's statistics come from one stats block (T0 <= 256: one atomicAdd onto zero).  Longer clips merge 256-row
blocks with fp64 atomics in an order that varies from call to call, so they are held to the bar only.

Interpolation bar: out = l0 a + l1 b with ATen's fp32 source positions (scale = f32(Tin) / f32(Tout), src =
fl(scale (t + 0.5) - 0.5) rounded once, as torch computes it, clamped at 0; i0, i1 = min(i0 + 1, Tin - 1); l1 =
f32(src - i0), l0 = f32(1 - l1)); two fp32 roundings of the weighted sum: 2^-23 (|l0 a| + |l1 b|).  torch's own
F.interpolate(mode='linear', align_corners=False) on the CPU must agree with the kernel within twice that bar (both
within the bar of the exact value): this pins the position rounding to the reference's, which matters at 100 s where
positions reach 5000 and one ulp of a position is 5e-4 of the interpolation weight.  Exact: Tout = Tin reproduces x.

LayerNorm bar, per element (a = x + pre in float64, n = ceil(C / 32) values per lane, mean / sd / rstd of a, dev = a -
mean, Ma = mean |a|):
  * the pre-add rounds: da <= u |a| (when pre is given);
  * the mean: lane sums of n values and the 5-level xor tree, then / C: dmean <= (n + 6) u Ma + mean da;
  * the two-pass variance: (n + 6) u var from the fmaf lane chains and the tree, 2 sd (max da + u max |dev|) from the
    rounded deviations, dmean^2; rstd = 1 / sqrtf(q / C + eps): 3 u plus half the variance's relative error over
    (var + eps);
  * the normalise / affine chain: |g| rstd (dmean + da + 2 u |dev|) + |g| |dev| rstd (e_rstd + 3 u) + u (|b| + |o|),
    + u |o + res| for the residual add (res = hi + lo exactly); ReLU does not grow it.
Input range (include/talkshow_b200.h): the row sum and the sum of squares are fp32, so |x| must stay below ~1e17.
Exact: mode 1's hi + lo is the mode-0 output bit for bit and hi has its 13 low bits clear; mode 6's planes are
h = fp16(o), l = fp16(o - h) of the fp32 o in y; repeat calls and an item alone vs inside a batch; the pad rows of the
output keep the caller's sentinels.

VQ argmin bar: the kernel's distance d_n = (xx + ee_n) - 2 dot_n with xx and dot_n 64-long fp32 FMA chains (gamma_64 =
64 u / (1 - 64 u) each), ee_n rounded once from an exact sum (u), and two more roundings: |d_n - d64_n| <= bar_n =
67 u (sum z^2 + sum e_n^2 + 2 sum |z| |e_n|).  So (a) d64(idx) <= min d64 + bar(idx) + bar(argmin) on every row;
(b) idx is the float64 argmin wherever every other code's distance exceeds the minimum by more than both bars; (c) idx
equals the oracle's torch fp32 vq_code_indices under the same condition; (d) exact duplicate codebook rows give the
lowest index.  Non-finite latents follow torch.argmin: a NaN distance wins, first such code.

Statistical bar: the RMS over the outputs of |error| / (per-element bar) is pinned per kernel and format at 4x the
largest value measured over the cases below on one H100 80GB HBM3 (700 W power limit); see RMS_BAR.  Every case prints
its statistics ("conv0 ..." / "interp ..." / "ln ..." / "vq ..." lines, pytest -s)."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import talkshow_oracle as O
from talkshow_b200 import _lib, synth

pytestmark = pytest.mark.gpu

TS_ERR_INVALID = 1
U = 2.0 ** -24
SENT = 1234.5
SENT16 = 0x5A5A
# RMS of |error| / (per-element bar), 4x the largest value measured on one H100 80GB HBM3 (700 W power limit)
# (700 W power limit), over the cases the RMS is checked on.  Largest measured: conv0 1.06e-2 in every format (DC plus
# a small signal, T0 701); interp 0.252 (B 1, Tin 49, Tout 48, C 1: the per-element bar is tight there, so this adds
# little); LayerNorm 0.243 in every format (magnitude 1e-4, variance below eps, C 33)
RMS_BAR = {"conv0": {0: 4 * 1.06e-2, 1: 4 * 1.06e-2, 6: 4 * 1.06e-2}, "interp": 4 * 0.252, "ln": {0: 4 * 0.243, 1: 4 * 0.243, 6: 4 * 0.243}}


@pytest.fixture(scope="module")
def eng():
    from talkshow_b200.engine import Engine

    torch.set_grad_enabled(False)
    e = Engine(0)
    yield e
    torch.cuda.synchronize()
    e.close()


def host(t):
    a = np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32))
    return a, a.ctypes.data_as(C.c_void_p)


def stats_line(kind, label, err, bar):
    r = err / bar
    rms, mx = float(r.pow(2).mean().sqrt()), float(r.max())
    print("%s %-40s rms %.3g max %.3g (err / bar)" % (kind, label, rms, mx))
    return rms


def fail_first(label, bad, got, ref, bar):
    i = tuple(bad.nonzero()[0].tolist())
    pytest.fail("%s: %d elements over the bar, first %s: got %.9g ref %.9g bar %.3g" % (
        label, int(bad.sum()), i, float(got[i]), float(ref[i]), float(bar[i])))


def gelu64(z):
    return 0.5 * z * (1 + torch.special.erf(z / math.sqrt(2)))


# ---- conv0 + GroupNorm + GELU ------------------------------------------------------------------------------------------
def c0_params(seed):
    gen = torch.Generator().manual_seed(seed)
    W = torch.randn(512, 1, 10, generator=gen) * 0.3
    g = 1 + 0.3 * torch.randn(512, generator=gen)
    b = 0.5 * torch.randn(512, generator=gen)
    return W, g, b


def c0_call(e, mode, wave, W, g, b):
    """-> (status, value [B,R,512] as float64 (R = T0 + (T0 & 1)), raw planes, launches)."""
    B, N = wave.shape
    T0 = (N - 10) // 5 + 1 if N >= 10 else 1
    R = T0 + (T0 & 1)
    y = hi = lo = None
    if mode == 0:
        y = torch.full((B, R, 512), SENT, device="cuda")
    elif mode == 1:
        hi = torch.full((B, R, 512), SENT, device="cuda")
        lo = hi.clone()
    else:
        hi = torch.full((B, R, 512), SENT16, dtype=torch.int16, device="cuda")
        lo = hi.clone()
    (Wn, Wp), (gn, gp), (bn, bp) = host(W), host(g), host(b)
    n0 = e.launches
    rc = e.L.ts_debug_conv0_gn(e.h, mode, _lib.ptr(wave), Wp, gp, bp, _lib.ptr(y), _lib.ptr(hi), _lib.ptr(lo), B, N, e._s())
    torch.cuda.synchronize()
    if mode == 0:
        v = y.double()
    elif mode == 1:
        v = (hi + lo).double()
    else:
        v = hi.view(torch.float16).double() + lo.view(torch.float16).double()
    return rc, v, (y, hi, lo), e.launches - n0


def c0_reference(wave, W, g, b):
    """float64: z (pre-GELU), out = GELU(z) and the per-element bar of the module docstring, each [B,T0,512]."""
    B, N = wave.shape
    T0 = (N - 10) // 5 + 1
    win = wave.double().cuda().unfold(1, 10, 5)[:, :T0]                     # [B, T0, 10]
    Wd = W.double().cuda().view(512, 10)
    y = win @ Wd.T
    S = win.abs() @ Wd.abs().T
    mean = y.mean(1, keepdim=True)
    var = (y - mean).pow(2).mean(1, keepdim=True)
    sd = var.sqrt()
    rstd = 1 / torch.sqrt(var + 1e-5)
    gg, bb = g.double().cuda().view(1, 1, 512), b.double().cuda().view(1, 1, 512)
    z = (y - mean) * rstd * gg + bb
    out = gelu64(z)
    D = 10 * U * S
    Dm = D.mean(1, keepdim=True)
    Dmax = D.amax(1, keepdim=True)
    dvar = 2 * sd * Dmax + Dmax ** 2 + 4 * 2.0 ** -53 * y.pow(2).mean(1, keepdim=True)
    e_r = 0.5 * dvar / (var + 1e-5) + U
    a = (y - mean).abs() * rstd
    dz = gg.abs() * rstd * (D + Dm + 2 * U * mean.abs()) + gg.abs() * a * (e_r + 4 * U) + U * (bb.abs() + z.abs())
    bar = 1.13 * dz + 2.0 ** -21 * z.abs() + 2.0 ** -22 * out.abs()
    return z, out, bar


def c0_check(mode, wave, W, g, b, v, label, rms=True):
    B, N = wave.shape
    T0 = (N - 10) // 5 + 1
    z, ref, bar = c0_reference(wave, W, g, b)
    if mode == 6:
        bar = bar + 2.0 ** -22 * ref.abs() + 2.0 ** -25
    got = v[:, :T0]
    assert torch.isfinite(got).all(), "%s: non-finite or unwritten outputs" % label
    err = (got - ref).abs()
    bad = err > bar
    if bad.any():
        fail_first(label, bad, got, ref, bar)
    if T0 & 1:
        assert torch.isnan(v[:, T0:]).all(), "%s: a tail row was written" % label
    st = stats_line("conv0", "%s m%d B %d T0 %d" % (label, mode, B, T0), err, bar)
    if rms:
        assert st <= RMS_BAR["conv0"][mode], "%s: RMS err / bar %.3g over %.3g" % (label, st, RMS_BAR["conv0"][mode])
    return got


def c0_wave(B, N, seed, kind="speech"):
    gen = torch.Generator().manual_seed(seed)
    if kind == "speech":
        return synth.synth_wave(B, N, seed=seed).float().contiguous()
    if kind == "silence":
        return torch.zeros(B, N)
    if kind == "dc":
        return torch.full((B, N), 0.37)
    if kind == "dc_signal":                                  # mean / std of y ~ 1e3: the E[y^2] - mean^2 cancellation
        return (1.0 + 1e-3 * torch.randn(B, N, generator=gen)).contiguous()
    if kind == "amp1e3":
        return (1e3 * synth.synth_wave(B, N, seed=seed).float()).contiguous()
    raise ValueError(kind)


C0_LEN = [10, 11, 12, 13, 14, 400, 401, 402, 403, 404, 5 * 62 + 10, 5 * 63 + 10, 5 * 64 + 10, 5 * 254 + 10, 5 * 255 + 10,
          5 * 256 + 10, 60 * 16000, 100 * 16000]
C0_IDS = [(m, N, B) for m in (6, 1, 0) for N in C0_LEN for B in ((1, 3, 7) if N <= 1290 else (1, 3) if N < 1600000 else (1,))]


@pytest.mark.parametrize("mode,N,B", C0_IDS, ids=["m%d-N%d-B%d" % p for p in C0_IDS])
def test_conv0_gn_lengths(eng, mode, N, B):
    """T0 = 1 (zero variance), every (N - 10) mod 5, the face's minimum of 400 samples, the apply (64) and stats (256)
    block edges, and 60 s / 100 s clips (hundreds of stats blocks merged by fp64 atomics)."""
    wave = c0_wave(B, N, seed=zlib.crc32(b"c0%d" % N) + B).cuda()
    W, g, b = c0_params(seed=N % 97)
    rc, v, _, n = c0_call(eng, mode, wave, W, g, b)
    assert rc == 0 and n == 3, eng.L.ts_last_error(eng.h)          # the NaN tail fill, the stats and the apply kernels
    c0_check(mode, wave, W, g, b, v, "lengths")


@pytest.mark.parametrize("mode", [6, 1, 0])
@pytest.mark.parametrize("kind", ["silence", "dc", "dc_signal", "amp1e3"])
def test_conv0_gn_signals(eng, mode, kind):
    """Silence and a constant wave give GELU(beta) at every t; DC plus a small signal and a x1e3 amplitude meet the bar."""
    for B, N in ((3, 400), (2, 5 * 700 + 13)):
        wave = c0_wave(B, N, seed=5, kind=kind).cuda()
        W, g, b = c0_params(seed=11)
        rc, v, _, _ = c0_call(eng, mode, wave, W, g, b)
        assert rc == 0
        got = c0_check(mode, wave, W, g, b, v, kind, rms=kind not in ("silence", "dc"))
        if kind in ("silence", "dc"):
            assert (got == got[:, :1]).all(), "%s: rows differ" % kind
            want = gelu64(b.double().cuda()).view(1, 1, 512)
            tol = 2.0 ** -21 * b.double().cuda().abs().view(1, 1, 512) + 2.0 ** -22 * want.abs() + (
                2.0 ** -22 * want.abs() + 2.0 ** -25 if mode == 6 else 0)
            assert ((got - want).abs() <= tol).all(), "%s: not GELU(beta)" % kind


def test_conv0_gn_exact(eng):
    """Where each clip's statistics come from one block (T0 <= 256): repeat calls, an item alone vs inside a batch of 7
    and perturbed samples past the last window give the same bits, and the three formats hold the same values."""
    W, g, b = c0_params(seed=3)
    for N in (5 * 255 + 10 + 4, 403, 14):
        wave = c0_wave(7, N, seed=N).cuda()
        T0 = (N - 10) // 5 + 1
        _, full, _, _ = c0_call(eng, 0, wave, W, g, b)
        _, again, _, _ = c0_call(eng, 0, wave, W, g, b)
        assert torch.equal(full.nan_to_num(7.0), again.nan_to_num(7.0)), N
        for i in (0, 3, 6):
            _, one, _, _ = c0_call(eng, 0, wave[i:i + 1].contiguous(), W, g, b)
            assert torch.equal(one[:, :T0], full[i:i + 1, :T0]), (N, i)
        used = 5 * (T0 - 1) + 10
        if used < N:
            w2 = wave.clone()
            w2[:, used:] = 1e6
            _, pert, _, _ = c0_call(eng, 0, w2, W, g, b)
            assert torch.equal(pert[:, :T0], full[:, :T0]), "N %d: samples past the last window were read" % N
        _, _, (_, hi, lo), _ = c0_call(eng, 1, wave, W, g, b)
        assert (hi[:, :T0].view(torch.int32) & 0x1FFF).eq(0).all()
        assert torch.equal((hi + lo)[:, :T0].double(), full[:, :T0]), N
        _, _, (_, h16, l16), _ = c0_call(eng, 6, wave, W, g, b)
        o = full[:, :T0].float().cpu().numpy()
        h = o.astype(np.float16)
        l = (o - h.astype(np.float32)).astype(np.float16)
        assert np.array_equal(h16[:, :T0].cpu().numpy().view(np.uint16), h.view(np.uint16)), N
        assert np.array_equal(l16[:, :T0].cpu().numpy().view(np.uint16), l.view(np.uint16)), N


def test_conv0_gn_refused_without_launch(eng):
    W, g, b = c0_params(seed=1)
    (_, Wp), (_, gp), (_, bp) = host(W), host(g), host(b)
    wave = torch.zeros(1, 400, device="cuda")
    y = torch.full((1, 78, 512), SENT, device="cuda")
    for mode, B, N, planes in ((2, 1, 400, False), (7, 1, 400, False), (0, 0, 400, False), (0, 1, 9, False),
                               (6, 1, 400, False), (1, 1, 400, False)):
        n0 = eng.launches
        rc = eng.L.ts_debug_conv0_gn(eng.h, mode, _lib.ptr(wave), Wp, gp, bp, _lib.ptr(y), None, None, B, N, eng._s())
        assert rc == TS_ERR_INVALID and eng.launches == n0 and (y == SENT).all(), (mode, B, N)
    assert eng.L.ts_debug_conv0_gn(eng.h, 0, _lib.ptr(wave), None, gp, bp, _lib.ptr(y), None, None, 1, 400, eng._s()) == TS_ERR_INVALID


# ---- interpolation -----------------------------------------------------------------------------------------------------
def interp_call(e, x, Tout, y=None):
    B, Tin, Cc = x.shape
    y = torch.full((B, Tout, Cc), SENT, device="cuda") if y is None else y
    n0 = e.launches
    rc = e.L.ts_debug_interp(e.h, _lib.ptr(x), _lib.ptr(y), B, Tin, Tout, Cc, e._s())
    torch.cuda.synchronize()
    return rc, y, e.launches - n0


def interp_reference(x, Tout):
    """float64 l0 a + l1 b with torch's fp32 positions, and the bar 2^-23 (|l0 a| + |l1 b|)."""
    Tin = x.shape[1]
    f32 = np.float32
    scale = f32(f32(Tin) / f32(Tout))
    t = np.arange(Tout, dtype=np.float32) + f32(0.5)
    src = (np.float64(scale) * t.astype(np.float64) - 0.5).astype(np.float32)     # exact in float64, rounded once
    src = np.maximum(src, f32(0))
    i0 = np.minimum(src.astype(np.int64), Tin - 1)
    i1 = np.where(i0 < Tin - 1, i0 + 1, i0)
    l1 = (src - i0.astype(np.float32)).astype(np.float32)
    l0 = (f32(1) - l1).astype(np.float32)
    xd = x.double()
    dev = xd.device
    A = torch.from_numpy(l0.astype(np.float64)).to(dev).view(1, -1, 1) * xd[:, torch.from_numpy(i0).to(dev)]
    Bv = torch.from_numpy(l1.astype(np.float64)).to(dev).view(1, -1, 1) * xd[:, torch.from_numpy(i1).to(dev)]
    return A + Bv, 2.0 ** -23 * (A.abs() + Bv.abs())


def interp_check(x, Tout, y, label):
    assert torch.isfinite(y).all(), "%s: non-finite or unwritten outputs" % label
    ref, bar = interp_reference(x, Tout)
    err = (y.double() - ref).abs()
    bad = err > bar
    if bad.any():
        fail_first(label, bad, y, ref, bar)
    tr = F.interpolate(x.cpu().permute(0, 2, 1), size=Tout, mode="linear", align_corners=False).permute(0, 2, 1)
    terr = (y.cpu().double() - tr.double()).abs()
    tbad = terr > 2 * bar.cpu()
    if tbad.any():
        fail_first(label + " vs torch CPU", tbad, y.cpu(), tr, 2 * bar.cpu())
    pos = bar > 0
    if pos.any():
        st = stats_line("interp", "%s B %d Tin %d Tout %d C %d" % (label, x.shape[0], x.shape[1], Tout, x.shape[2]),
                        err[pos], bar[pos])
        assert st <= RMS_BAR["interp"], "%s: RMS err / bar %.3g" % (label, st)


@pytest.mark.parametrize("Tin", [1, 2, 49, 50])
@pytest.mark.parametrize("Cc", [512, 1, 3])
def test_interp_shapes(eng, Tin, Cc):
    """Down- and upsampling around every Tin, one and three channels as well as the face's 512, B = 1 and 5."""
    for Tout in sorted({1, max(1, Tin - 1), Tin, Tin + 1, 2 * Tin + 1}):
        for B in (1, 5):
            gen = torch.Generator().manual_seed(zlib.crc32(b"in%d-%d-%d" % (Tin, Tout, Cc)) + B)
            x = torch.randn(B, Tin, Cc, generator=gen).cuda()
            rc, y, n = interp_call(eng, x, Tout)
            assert rc == 0 and n == 2, eng.L.ts_last_error(eng.h)   # the staging fill and the interpolation
            interp_check(x, Tout, y, "shapes")
            if Tout == Tin:
                assert torch.equal(y, x), "Tout = Tin is not the identity"


def w2v_frames(N):
    T = (N - 10) // 5 + 1
    for k in (3, 3, 3, 3, 2, 2):
        T = (T - k) // 2 + 1
    return T


@pytest.mark.parametrize("sec", [1, 10, 100])
def test_interp_face_ratio(eng, sec):
    """The face's own 50 -> 30 fps ratio at 1 s, 10 s and 100 s (Tin 4999: positions reach 5000)."""
    Tin, Tout = w2v_frames(sec * 16000), sec * 30
    B = 2 if sec < 100 else 1
    x = torch.randn(B, Tin, 512, generator=torch.Generator().manual_seed(sec)).cuda()
    rc, y, _ = interp_call(eng, x, Tout)
    assert rc == 0
    interp_check(x, Tout, y, "face %d s" % sec)


def test_interp_refused(eng):
    x = torch.zeros(1, 8, 4, device="cuda")
    y = torch.full((1, 5, 4), SENT, device="cuda")
    for B, Tin, Tout, Cc in ((0, 8, 5, 4), (1, 0, 5, 4), (1, 8, 0, 4), (1, 8, 5, 0)):
        n0 = eng.launches
        assert eng.L.ts_debug_interp(eng.h, _lib.ptr(x), _lib.ptr(y), B, Tin, Tout, Cc, eng._s()) == TS_ERR_INVALID
        assert eng.launches == n0 and (y == SENT).all()
    assert eng.L.ts_debug_interp(eng.h, None, _lib.ptr(y), 1, 8, 5, 4, eng._s()) == TS_ERR_INVALID


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------
class DebugLN(C.Structure):
    _fields_ = [(f, C.c_int32) for f in ("mode", "B", "T", "C", "has_pre", "has_res", "act", "x_split", "res_split",
                                         "y_split")]


def ln_call(e, mode, x, g, b, pre=None, res=None, act=0, x_split=0, res_split=0, y_split=0):
    """-> (status, y or None, hi, lo, launches); output buffers [B, T + 2, C] start as sentinels."""
    B, T, Cc = x.shape
    y = hi = lo = None
    if not y_split or mode == 6:
        y = torch.full((B, T + 2, Cc), SENT, device="cuda")
    if y_split:
        hi = (torch.full((B, T + 2, Cc), SENT16, dtype=torch.int16, device="cuda") if mode == 6
              else torch.full((B, T + 2, Cc), SENT, device="cuda"))
        lo = hi.clone()
    a = DebugLN(mode, B, T, Cc, pre is not None, res is not None, act, x_split, res_split, y_split)
    (_, gp), (_, bp) = host(g), host(b)
    n0 = e.launches
    rc = e.L.ts_debug_layernorm(e.h, C.byref(a), _lib.ptr(x), _lib.ptr(pre), _lib.ptr(res), gp, bp, _lib.ptr(y),
                                _lib.ptr(hi), _lib.ptr(lo), e._s())
    torch.cuda.synchronize()
    return rc, y, hi, lo, e.launches - n0


def ln_reference(x, g, b, pre, res, act):
    """float64 output and the per-element bar of the module docstring."""
    Cc = x.shape[2]
    n = -(-Cc // 32)
    a = x.double() + (pre.double() if pre is not None else 0)
    da = U * a.abs() if pre is not None else torch.zeros_like(a)
    mean = a.mean(2, keepdim=True)
    dev = a - mean
    var = dev.pow(2).mean(2, keepdim=True)
    sd = var.sqrt()
    rstd = 1 / torch.sqrt(var + 1e-5)
    gg, bb = g.double().cuda().view(1, 1, -1), b.double().cuda().view(1, 1, -1)
    o = dev * rstd * gg + bb
    dmean = (n + 6) * U * a.abs().mean(2, keepdim=True) + da.mean(2, keepdim=True)
    dvar = (n + 6) * U * var + 2 * sd * (da.amax(2, keepdim=True) + U * dev.abs().amax(2, keepdim=True)) + dmean ** 2
    e_r = 3 * U + 0.5 * dvar / (var + 1e-5)
    bar = gg.abs() * rstd * (dmean + da + 2 * U * dev.abs()) + gg.abs() * dev.abs() * rstd * (e_r + 3 * U) + U * (bb.abs() + o.abs())
    if res is not None:
        o = o + res.double()
        bar = bar + U * o.abs()
    if act == 1:
        o = o.clamp_min(0)
    return o, bar


def ln_value(mode, y_split, y, hi, lo):
    """The output value [B, T + 2, C] and a check that every buffer's pad rows still hold the caller's sentinels."""
    for t in (y, hi, lo):
        if t is not None:
            s = SENT16 if t.dtype == torch.int16 else SENT
            assert (t[:, 0] == s).all() and (t[:, -1] == s).all(), "a pad row was written"
    if y_split and mode != 6:
        return hi + lo
    return y


def ln_check(mode, x, g, b, pre, res, act, out, label, rms=True):
    B, T, Cc = x.shape
    got = out[:, 1:T + 1].double()
    assert torch.isfinite(got).all(), "%s: non-finite or unwritten outputs" % label
    ref, bar = ln_reference(x, g, b, pre, res, act)
    err = (got - ref).abs()
    bad = err > bar
    if bad.any():
        fail_first(label, bad, got, ref, bar)
    st = stats_line("ln", "%s m%d B %d T %d C %d" % (label, mode, B, T, Cc), err, bar)
    if rms:
        assert st <= RMS_BAR["ln"][mode], "%s: RMS err / bar %.3g over %.3g" % (label, st, RMS_BAR["ln"][mode])


# the flag combinations face_run uses: hn / hcur (plain, split output), encoder LN (pre-add), first_net (residual +
# ReLU, split residual), decoder (ReLU), and a 3xTF32 input
COMBOS = {"plain": dict(), "pre": dict(pre=True), "res_relu": dict(res=True, act=1), "res_split_relu": dict(res=True, act=1, res_split=1),
          "relu": dict(act=1), "x_split": dict(x_split=1, res=True, res_split=1)}


def ln_inputs(B, T, Cc, seed, kind="normal"):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, Cc, generator=gen)
    if kind == "const":
        x = torch.randn(B, T, 1, generator=gen).expand(B, T, Cc).contiguous()
    elif kind == "mean1e4":
        x = 1e4 + 1e-2 * x
    elif kind == "mag1e-4":
        x = 1e-4 * x
    elif kind == "mag1e15":
        x = 1e15 * x
    pre = torch.randn(B, T, Cc, generator=gen) * x.abs().mean()
    res = torch.randn(B, T, Cc, generator=gen)
    g = 1 + 0.3 * torch.randn(Cc, generator=gen)
    b = 0.2 * torch.randn(Cc, generator=gen)
    return x.cuda(), pre.cuda(), res.cuda(), g, b


def ln_run(e, mode, combo, x, pre, res, g, b, y_split, label, rms=True):
    f = COMBOS[combo]
    p = pre if f.get("pre") else None
    r = res if f.get("res") else None
    rc, y, hi, lo, n = ln_call(e, mode, x, g, b, pre=p, res=r, act=f.get("act", 0), x_split=f.get("x_split", 0),
                               res_split=f.get("res_split", 0), y_split=y_split)
    assert rc == 0, e.L.ts_last_error(e.h)
    out = ln_value(mode, y_split, y, hi, lo)
    ln_check(mode, x, g, b, p, r, f.get("act", 0), out, "%s %s ys%d" % (label, combo, y_split), rms=rms)
    return y, hi, lo, out


LN_BT = [(1, 1), (1, 7), (2, 4), (3, 3), (4, 250)]


@pytest.mark.parametrize("mode", [6, 1, 0])
@pytest.mark.parametrize("Cc", [64, 256, 512, 768, 1, 33, 100, 767])
def test_layernorm_widths(eng, mode, Cc):
    """Production and odd widths, 1 / 7 / 8 / 9 / 1000 rows (8 warps per block and the early exit), every flag
    combination and both output forms; the split outputs are the plain output's bits."""
    for B, T in LN_BT:
        x, pre, res, g, b = ln_inputs(B, T, Cc, seed=zlib.crc32(b"ln%d-%d-%d" % (Cc, B, T)))
        for combo in COMBOS:
            plain = ln_run(eng, mode, combo, x, pre, res, g, b, 0, "widths")[3]
            y, hi, lo, out = ln_run(eng, mode, combo, x, pre, res, g, b, 1, "widths")
            if mode == 6:
                assert torch.equal(y, plain)
                o = y[:, 1:T + 1].cpu().numpy()
                h = o.astype(np.float16)
                l = (o - h.astype(np.float32)).astype(np.float16)
                assert np.array_equal(hi[:, 1:T + 1].cpu().numpy().view(np.uint16), h.view(np.uint16))
                assert np.array_equal(lo[:, 1:T + 1].cpu().numpy().view(np.uint16), l.view(np.uint16))
                assert (hi[:, 0] == SENT16).all() and (lo[:, T + 1] == SENT16).all()
            else:
                assert (hi[:, 1:T + 1].view(torch.int32) & 0x1FFF).eq(0).all()
                assert torch.equal(out[:, 1:T + 1], plain[:, 1:T + 1]), (combo, "hi + lo differs from the plain output")


@pytest.mark.parametrize("mode", [6, 1, 0])
@pytest.mark.parametrize("kind", ["const", "mean1e4", "mag1e-4", "mag1e15"])
def test_layernorm_inputs(eng, mode, kind):
    """Constant rows, mean 1e4 with std 1e-2, magnitude 1e-4 (variance below eps) and 1e15 (inside the fp32 range of
    the sum of squares)."""
    for Cc in (768, 256, 33):
        x, pre, res, g, b = ln_inputs(3, 5, Cc, seed=zlib.crc32(kind.encode()) + Cc, kind=kind)
        for combo in ("plain", "pre", "res_relu", "x_split"):
            ln_run(eng, mode, combo, x, pre, res, g, b, 1 if mode == 6 else 0, kind, rms=kind != "mean1e4")


def test_layernorm_exact(eng):
    """Repeat calls and an item alone vs inside a batch of 7 give the same bits."""
    x, pre, res, g, b = ln_inputs(7, 33, 768, seed=9)
    for mode in (6, 1, 0):
        for combo in ("pre", "res_split_relu"):
            full = ln_run(eng, mode, combo, x, pre, res, g, b, 0, "exact")[3]
            again = ln_run(eng, mode, combo, x, pre, res, g, b, 0, "exact")[3]
            assert torch.equal(full, again)
            for i in (0, 3, 6):
                one = ln_run(eng, mode, combo, x[i:i + 1].contiguous(), pre[i:i + 1].contiguous(), res[i:i + 1].contiguous(),
                             g, b, 0, "exact")[3]
                assert torch.equal(one, full[i:i + 1]), (mode, combo, i)


def test_layernorm_refused_without_launch(eng):
    x, pre, res, g, b = ln_inputs(1, 4, 769, seed=1)
    (_, gp), (_, bp) = host(g), host(b)
    y = torch.full((1, 6, 769), SENT, device="cuda")
    bad = [DebugLN(0, 1, 4, 769, 0, 0, 0, 0, 0, 0), DebugLN(2, 1, 4, 64, 0, 0, 0, 0, 0, 0), DebugLN(0, 0, 4, 64, 0, 0, 0, 0, 0, 0),
           DebugLN(0, 1, 4, 64, 0, 0, 2, 0, 0, 0), DebugLN(0, 1, 4, 64, 1, 0, 0, 0, 0, 0), DebugLN(0, 1, 4, 64, 0, 1, 0, 0, 0, 0),
           DebugLN(1, 1, 4, 64, 0, 0, 0, 0, 0, 1), DebugLN(6, 1, 4, 64, 0, 0, 0, 0, 0, 1)]
    for a in bad:
        n0 = eng.launches
        rc = eng.L.ts_debug_layernorm(eng.h, C.byref(a), _lib.ptr(x), None, None, gp, bp, _lib.ptr(y), None, None, eng._s())
        assert rc == TS_ERR_INVALID and eng.launches == n0 and (y == SENT).all(), [getattr(a, f) for f, _ in a._fields_]


# ---- VQ argmin ---------------------------------------------------------------------------------------------------------
def vq_call(e, cb, z):
    R = z.shape[0]
    idx = torch.full((R,), -7, dtype=torch.int64, device="cuda")
    cbn, cbp = host(cb)
    n0 = e.launches
    rc = e.L.ts_debug_vq_argmin(e.h, cbp, cb.shape[0], _lib.ptr(z), _lib.ptr(idx), R, e._s())
    torch.cuda.synchronize()
    return rc, idx, e.launches - n0


def vq_reference(cb, z):
    """float64 distances [R, ncodes] and the per-code bars."""
    zd, ed = z.double().cuda(), cb.double().cuda()
    zz, ee = zd.pow(2).sum(1, keepdim=True), ed.pow(2).sum(1).view(1, -1)
    d = zz + ee - 2 * zd @ ed.T
    bar = 67 * U * (zz + ee + 2 * zd.abs() @ ed.abs().T)
    return d, bar


def vq_check(cb, z, idx, label):
    ncodes = cb.shape[0]
    assert ((idx >= 0) & (idx < ncodes)).all(), "%s: index out of range" % label
    d, bar = vq_reference(cb, z)
    r = torch.arange(z.shape[0], device=idx.device)
    dmin, amin = d.min(1)
    got_d, got_b = d[r, idx], bar[r, idx]
    ok_a = got_d <= dmin + got_b + bar[r, amin]
    assert ok_a.all(), "%s: (a) %d rows pick a code beyond both bars" % (label, int((~ok_a).sum()))
    lower = d - bar
    lower[r, amin] = float("inf")
    clear = lower.min(1).values > dmin + bar[r, amin]          # every other code is out of reach
    assert torch.equal(idx[clear], amin[clear]), "%s: (b) %d clear rows differ from the float64 argmin" % (
        label, int((idx[clear] != amin[clear]).sum()))
    oracle = O.vq_code_indices({"vq_layer.embeddings": cb.float().cpu()}, z.float().cpu()).to(idx.device)
    assert torch.equal(idx[clear], oracle[clear]), "%s: (c) clear rows differ from the oracle" % label
    worst = float(((got_d - dmin) / (got_b + bar[r, amin])).max())
    print("vq %-40s R %5d ncodes %4d: %d / %d rows clear, %d rows differ from float64, worst (d - min) / bars %.3g" % (
        label, z.shape[0], ncodes, int(clear.sum()), z.shape[0], int((idx != amin).sum()), worst))


def vq_data(R, ncodes, scale, seed, clustered=False):
    gen = torch.Generator().manual_seed(seed)
    cb = torch.randn(ncodes, 64, generator=gen)
    if clustered:                                  # 8 centres, codes within 1e-3 of them: near-ties everywhere
        cb = torch.randn(8, 64, generator=gen)[torch.arange(ncodes) % 8] + 1e-3 * cb
    z = cb[torch.randint(0, ncodes, (R,), generator=gen)] + 0.5 * torch.randn(R, 64, generator=gen)
    return (cb * scale).contiguous(), (z * scale).contiguous().cuda()


VQ_IDS = [(n, R, s) for n in (1, 2, 255, 256, 257, 1000, 1024, 2048) for R in (1, 19200) for s in (1e-3, 1.0, 1e3)]


@pytest.mark.parametrize("ncodes,R,scale", VQ_IDS, ids=["n%d-R%d-s%g" % p for p in VQ_IDS])
def test_vq_argmin_sizes(eng, ncodes, R, scale):
    """Every stride / warp edge of the 256-thread search, one row and 19200 rows, and scales where |z|^2 dwarfs the
    spread of the distances."""
    cb, z = vq_data(R, ncodes, scale, seed=zlib.crc32(b"vq%d-%d" % (ncodes, R)))
    rc, idx, n = vq_call(eng, cb, z)
    assert rc == 0 and n == 2, eng.L.ts_last_error(eng.h)       # the staging fill and the argmin
    vq_check(cb, z, idx, "sizes s %g" % scale)


@pytest.mark.parametrize("ncodes", [257, 2048])
def test_vq_argmin_near_ties(eng, ncodes):
    """Clustered codebooks (near-ties in every row) and latents equal to codebook rows (distance 0 against one code)."""
    cb, z = vq_data(4096, ncodes, 1.0, seed=ncodes, clustered=True)
    rc, idx, _ = vq_call(eng, cb, z)
    assert rc == 0
    vq_check(cb, z, idx, "clustered")
    cb, _ = vq_data(1, ncodes, 1.0, seed=ncodes + 1)
    pick = torch.randint(0, ncodes, (512,), generator=torch.Generator().manual_seed(1))
    z = cb[pick].contiguous().cuda()
    rc, idx, _ = vq_call(eng, cb, z)
    assert rc == 0 and torch.equal(idx.cpu(), pick), "z = codebook row: not that row's code"
    vq_check(cb, z, idx, "z = codebook row")


def test_vq_argmin_duplicates(eng):
    """Exact duplicate codebook rows in one thread (5, 261, 1029), another warp (300) and the last code (2047): the
    lowest index wins."""
    cb, _ = vq_data(1, 2048, 1.0, seed=5)
    dup = [5, 261, 300, 1029, 2047]
    for order in (dup, dup[::-1]):
        c = cb.clone()
        c[order] = cb[order[0]]
        z = (c[5] + 1e-3 * torch.randn(64, generator=torch.Generator().manual_seed(2))).view(1, 64).repeat(33, 1).cuda()
        rc, idx, _ = vq_call(eng, c, z)
        assert rc == 0 and (idx == 5).all(), idx
    c = cb.clone()
    c[[300, 1029, 2047]] = cb[300]
    z = c[300].view(1, 64).cuda()
    rc, idx, _ = vq_call(eng, c, z)
    assert rc == 0 and int(idx[0]) == 300


def test_vq_argmin_non_finite(eng):
    """A latent with a NaN gets code 0; one +inf component against a codebook whose component is negative for codes
    < j and positive at j gives distances +inf for n < j and NaN at j, so the first NaN code j, as the oracle's
    torch.argmin; every index is in range."""
    ncodes = 1000
    cb, z = vq_data(64, ncodes, 1.0, seed=8)
    z = z.clone()
    z[3, 17] = float("nan")
    z[10] = float("nan")
    rc, idx, _ = vq_call(eng, cb, z)
    assert rc == 0 and ((idx >= 0) & (idx < ncodes)).all()
    assert int(idx[3]) == 0 and int(idx[10]) == 0
    finite = torch.isfinite(z).all(1)
    vq_check(cb, z[finite].contiguous(), idx[finite], "finite rows beside NaN rows")
    for j in (0, 1, 300, 999):
        c = cb.clone()
        c[:, 40] = -c[:, 40].abs() - 0.1
        c[j, 40] = 0.5
        zi = z[:1].clone()
        zi[0, 40] = float("inf")
        rc, idx, _ = vq_call(eng, c, zi)
        oracle = O.vq_code_indices({"vq_layer.embeddings": c}, zi.cpu())
        assert rc == 0 and int(idx[0]) == j == int(oracle[0]), (j, int(idx[0]), int(oracle[0]))


def test_vq_argmin_refused(eng):
    cb, z = vq_data(4, 8, 1.0, seed=1)
    (_, cbp) = host(cb)
    idx = torch.full((4,), -7, dtype=torch.int64, device="cuda")
    for n, R in ((0, 4), (8, 0)):
        assert eng.L.ts_debug_vq_argmin(eng.h, cbp, n, _lib.ptr(z), _lib.ptr(idx), R, eng._s()) == TS_ERR_INVALID
    assert eng.L.ts_debug_vq_argmin(eng.h, None, 8, _lib.ptr(z), _lib.ptr(idx), 4, eng._s()) == TS_ERR_INVALID
    assert (idx == -7).all()


# ---- end to end: a NaN frame in one clip of a batch --------------------------------------------------------------------
def test_vq_encode_score_nan_frame(ckpts):
    """ts_vq_encode (with e_out) and ts_vq_score on a batch where clip 1 has a NaN frame: every index is in range, the
    other clips' indices, embeddings and clip_out are the bits of those clips scored alone, and on the rows the NaN
    cannot reach the NaN clip matches the oracle.  (The engine's ReLU maps NaN to 0 where torch.relu keeps it, so
    inside the encoder the NaN frame does not reach the latents: the rows it touches get finite codes.)"""
    from talkshow_b200.engine import Engine

    e = Engine(0)
    try:
        sd = ckpts["vq"]["g_body"]
        e.load_vq(0, sd)
        poses = synth.synth_poses(3, 96, seed=77)[:, O.C_INDEX_3D].permute(0, 2, 1)[..., :39].contiguous()
        poses[1, 50] = float("nan")
        ncodes = sd["vq_layer.embeddings"].shape[0]
        idx, emb = e.vq_encode(0, poses, want_e=True)
        sidx, clip, _ = e.vq_score(0, poses)
        assert ((idx >= 0) & (idx < ncodes)).all() and torch.equal(idx, sidx)
        _, ref = O.vq_encode(sd, poses)
        reach = torch.zeros(idx.shape[1], dtype=torch.bool)
        reach[4:21] = True      # latent rows whose receptive field (frames 4r - 25 .. 4r + 28) holds frame 50: 6 .. 18
        assert torch.equal(idx[1, ~reach].cpu(), ref[1, ~reach])
        for b in (0, 2):
            one = poses[b:b + 1].contiguous()
            i1, e1 = e.vq_encode(0, one, want_e=True)
            si1, c1, _ = e.vq_score(0, one)
            assert torch.equal(i1, idx[b:b + 1]) and torch.equal(e1, emb[b:b + 1]) and torch.equal(c1, clip[b:b + 1]), b
            assert torch.equal(i1.cpu(), ref[b:b + 1])
        print("vq end to end: NaN clip indices %s" % idx[1].tolist())
    finally:
        torch.cuda.synchronize()
        e.close()
