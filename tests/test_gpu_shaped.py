"""GPU (-m gpu): logit shaping of the body prior (repetition penalty and code bias; ts_pixelcnn_sample_shaped,
ts_body_sample_shaped) on every sampler executor of test_gpu_seeded.CONFIGS and on the 6-D prior, with explicit noise
and with seeds.

Pinned bit for bit: theta 1 without a bias, and a bias of zeros, draw what ts_pixelcnn_sample_clips draws (codes, log p,
keep sizes); a mixed batch equals each clip alone and each clip's setting run as a scalar call; the reference fixture's
codes and keep sizes (tests/golden/shaped.npz); the oracle's shaped draw (tests/oracle_shaped.py) on the engine's own
raw logits, anchors and a pre_latents prefix included; a banned code is never drawn.  Log p equals -nll of the
teacher-forced scorer on the drawn codes within the tolerance of the anchored tests.  Cluster-executor log p of separate
calls is compared at 1e-5 (the open issue of DESIGN §3d), everything else bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from talkshow_b200 import _lib, synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_nucleus as ON  # noqa: E402
import oracle_sampling as OSM  # noqa: E402
import oracle_shaped as OSH  # noqa: E402
from test_gpu_clip_ctl import GROUPS, SHAPES, SOURCES, _equal, _gen, _per_clip, _skip_tile, _tol  # noqa: E402
from test_gpu_seeded import CONFIGS, _aud, _engine, _seeds, config, eng, six  # noqa: E402,F401

pytestmark = pytest.mark.gpu
# the shaping clip b cycles through (penalty, window); with GROUPS' four controls this gives every pairing over 12 clips
SHAPING = [(1.0, 8), (1.5, 1), (2.0, 4), (3.0, 100000), (1.3, 8), (2.0, 8)]


def _shaping(B):
    return dict(repetition_penalty=[SHAPING[b % len(SHAPING)][0] for b in range(B)],
                repetition_window=[SHAPING[b % len(SHAPING)][1] for b in range(B)])


def _ban(B, seed):
    """a bias [B,2,2048]: 512 banned codes per row, a N(0, 1) bias elsewhere on odd clips"""
    g = torch.Generator().manual_seed(seed)
    bias = torch.zeros(B, 2, 2048)
    bias[1::2] = torch.randn(bias[1::2].shape, generator=g)
    banned = torch.rand(B, 2, 2048, generator=g).argsort(-1)[..., :512]
    bias.scatter_(-1, banned, float("-inf"))
    return bias


def _check_identity(e, ck, B, T, src, tol, what, seed):
    aud, label = _aud(ck, B, T, seed)
    seeds = _seeds(B, seed)
    noise = e.sampler_noise(seeds, T).cpu()
    pc = _per_clip(B)
    ref = _gen(e, aud, label, src, noise, seeds, **pc)
    # theta 1 on the clips beside penalised ones: their draws run the shaped kernels and equal the per-clip call
    sh = _shaping(B)
    got = _gen(e, aud, label, src, noise, seeds, **pc, **sh)
    idx = [b for b in range(B) if sh["repetition_penalty"][b] == 1.0]
    _equal([x[idx] for x in got], [x[idx] for x in ref], (what, "theta 1"), tol)
    # a bias of zeros on every clip: every draw shaped, nothing changed
    zero = _gen(e, aud, label, src, noise, seeds, code_bias=torch.zeros(2, 2048), **pc)
    _equal(zero, ref, (what, "zero bias"), tol)
    # a mixed batch equals each clip's setting as a scalar call and each clip alone
    bias = _ban(B, seed)
    got = _gen(e, aud, label, src, noise, seeds, code_bias=bias, **pc, **sh)
    for b in sorted({0, 3, B - 1} & set(range(B))):
        s = GROUPS[b % len(GROUPS)]
        t, w = SHAPING[b % len(SHAPING)]
        one = _gen(e, aud[b:b + 1], label[b:b + 1], src, noise[:, b:b + 1], seeds[b:b + 1], sampled=s["temperature"] > 0,
                   repetition_penalty=t, repetition_window=w, code_bias=bias[b], **s)
        _equal([x[b:b + 1] for x in got], one, (what, "alone", b), tol)
        scal = _gen(e, aud, label, src, noise, seeds, sampled=s["temperature"] > 0, repetition_penalty=t,
                    repetition_window=w, code_bias=bias, **s)
        _equal([x[b:b + 1] for x in got], [x[b:b + 1] for x in scal], (what, "scalar", b), tol)
    codes = got[0]
    assert not (bias.gather(-1, codes.transpose(1, 2)) == float("-inf")).any(), (what, "banned code drawn")


@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_identity_and_mixed_batch(eng, ckpts, config, B, T, src):
    _skip_tile(config, B)
    _check_identity(eng, ckpts["pixel"], B, T, src, _tol(config), (config, B, T, src), 700 + B)


@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("mb", ["4", "8"])
def test_identity_and_mixed_batch_6d(six, monkeypatch, mb, B, T, src):
    e, ck, _ = six
    monkeypatch.setenv("TS_PIX3_MB", mb)
    _check_identity(e, ck, B, T, src, 1e-5, ("6d", mb, B, T, src), 800 + B)


def _fixture_args(z, case):
    s = z["settings"].tolist()
    B = len(s)
    t, k, p, m, th, w = (list(c) for c in zip(*s))
    return B, dict(temperature=t, top_k=[int(x) for x in k], top_p=p, min_p=m, repetition_penalty=th,
                   repetition_window=[int(x) for x in w], code_bias=torch.from_numpy(z["bias_%s" % case]), want_kept=True)


@pytest.mark.parametrize("case", ["3d", "pre", "6d"])
def test_reference_fixture(eng, six, case):
    z = np.load(os.path.join(GOLDEN, "shaped.npz"))
    e = six[0] if case == "6d" else eng
    B, kw = _fixture_args(z, case)
    mfcc = torch.from_numpy(z["mfcc_%s" % case]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    noise = OSM.reference_noise(int(z["seed_%s" % case]), 2 * T, B)
    label = torch.full((B,), int(z["label_%s" % case]))
    if case == "pre":
        pre = torch.from_numpy(z["pre_%s" % case])
        mpre = torch.from_numpy(z["mfcc_pre_%s" % case]).repeat(B, 1, 1)
        aud = torch.cat([e.audio_encode(mpre), e.audio_encode(mfcc)], 2)
        codes, kept = e.pixelcnn_generate(aud, label, noise, T=T, pre_latents=pre, **kw)
    else:
        codes, _, kept = e.body_generate(mfcc, label, noise, **kw)
    assert torch.equal(codes.cpu(), torch.from_numpy(z["codes_%s" % case]))
    assert torch.equal(kept.cpu(), torch.from_numpy(z["kept_%s" % case]))


def _oracle_on_logits(codes, kept, logits, noise, pre, anchors, pc, sh, bias, what):
    """every sampled draw of the engine equals the oracle's shaped draw on the engine's raw logits and codes; draws whose
    nucleus or min-p keep set lies within 1e-5 of changing are skipped (the margin rule of the nucleus tests)"""
    B, T = codes.shape[:2]
    x = torch.cat([pre, codes], 1) if pre is not None else codes
    T0 = x.shape[1] - T
    n = 0
    for i in range(T):
        for j in range(2):
            lg = logits[2 * i + j]
            for b in range(B):
                if anchors is not None and anchors[b, i, j] >= 0:
                    assert codes[b, i, j] == anchors[b, i, j] and kept[b, i, j] == 0, (what, b, i, j)
                    continue
                t, k, p, m = (pc[key][b] for key in ("temperature", "top_k", "top_p", "min_p"))
                th, w = sh["repetition_penalty"][b], sh["repetition_window"][b]
                s = OSH.shape(lg[b], x[b, max(0, T0 + i - w):T0 + i, j], th, bias[b, j])[None]
                if t > 0 and (p < 1.0 or m > 0.0):
                    _, mp, mm = ON.keep_mask(s, t, k, p, m, return_margin=True)
                    if min(float(mp[0]), float(mm[0])) < 1e-5:
                        continue
                code, kn = OSH.draw(s, None if t == 0 else noise[2 * i + j][b:b + 1], t, k, p, m)
                assert int(code[0]) == int(codes[b, i, j]) and int(kn[0]) == int(kept[b, i, j]), (what, b, i, j)
                n += 1
    assert n >= B * T


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_oracle_on_engine_logits_with_anchors_and_pre_latents(eng, ckpts, config):
    B, T0, T = 12, 6, 16
    ck = ckpts["pixel"]
    aud, label = _aud(ck, B, T0 + T, 41)
    seeds = _seeds(B, 41)
    noise = eng.sampler_noise(seeds, T, T0).cpu()
    pre = torch.randint(0, 2048, (B, T0, 2), generator=torch.Generator().manual_seed(42))
    pre[:, -3:] = pre[:, -4:-3]
    anchors = torch.full((B, T, 2), -1, dtype=torch.int64)
    anchors[:, 3:5, 0] = torch.randint(0, 2048, (B, 2), generator=torch.Generator().manual_seed(43))
    pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, 44)
    codes, logits, logp, kept = (x.cpu() for x in eng.pixelcnn_generate(
        aud, label, noise, T=T, pre_latents=pre, want_logits=True, want_logp=True, want_kept=True, anchors=anchors,
        code_bias=bias, **pc, **sh))
    _oracle_on_logits(codes, kept, logits, noise, pre, anchors, pc, sh, bias, config)
    # log p is that of the raw prior: -nll of the teacher-forced scorer on the drawn codes
    full = torch.cat([pre, codes], 1)
    nll = eng.pixelcnn_score(aud, label, full).cpu()[:, T0:]
    assert (logp + nll).abs().mean() <= 2.5e-5 and (logp + nll).abs().max() <= 1e-4, config


def test_oracle_on_engine_logits_6d(six, monkeypatch):
    e, ck, _ = six
    B, T = 12, 10
    aud, label = _aud(ck, B, T, 45)
    seeds = _seeds(B, 45)
    noise = e.sampler_noise(seeds, T).cpu()
    pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, 46)
    for mb in ("4", "8"):
        monkeypatch.setenv("TS_PIX3_MB", mb)
        codes, logits, kept = (x.cpu() for x in e.pixelcnn_generate(aud, label, noise, want_logits=True, want_kept=True,
                                                                     code_bias=bias, **pc, **sh))
        _oracle_on_logits(codes, kept, logits, noise, None, None, pc, sh, bias, ("6d", mb))


def test_style_and_body_generate(eng, six):
    for e in (eng, six[0]):
        B, M = 12, 120
        mfcc = synth.synth_mfcc(B, M, seed=81)
        label = torch.arange(B) % 4
        seeds = _seeds(B, 81)
        w = torch.rand(B, 4, generator=torch.Generator().manual_seed(82)) + 0.1
        style = w / w.sum(-1, keepdim=True)
        pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, 83)
        codes, poses, logp = (x.cpu() for x in e.body_generate(mfcc, None, None, seeds=seeds, want_logp=True, style=style,
                                                               code_bias=bias, **pc, **sh))
        for b in (0, 3, 7):
            s = GROUPS[b % len(GROUPS)]
            t, win = SHAPING[b % len(SHAPING)]
            rc, rp, rl = (x.cpu() for x in e.body_generate(mfcc[b:b + 1], None, None, want_logp=True, style=style[b:b + 1],
                                                             seeds=seeds[b:b + 1] if s["temperature"] > 0 else None,
                                                             repetition_penalty=t, repetition_window=win, code_bias=bias[b],
                                                             **s))
            assert torch.equal(codes[b:b + 1], rc) and torch.equal(poses[b:b + 1], rp), b
            assert (logp[b:b + 1] - rl).abs().max() <= (1e-5 if e is six[0] else 0.0), b


def test_c_abi(eng, ckpts):
    from talkshow_b200.engine import CLIP_SHAPE

    B, T = 4, 6
    aud, label = _aud(ckpts["pixel"], B, T, 91)
    aud, label = aud.cuda(), label.cuda()
    seeds = _seeds(B, 91).cuda()
    noise = eng.sampler_noise(seeds, T)
    L, h, p = eng.L, eng.h, _lib.ptr
    s = _lib.stream_ptr(eng.device)

    def sample(noise_, seeds_, shape, bias):
        out = torch.empty(B, T, 2, dtype=torch.int64, device=eng.device)
        n0 = eng.launches
        rc = L.ts_pixelcnn_sample_shaped(h, p(aud), p(label), None, 4, p(noise_), p(seeds_), None, p(out), None, B, T, None,
                                         0, None, None, shape, p(bias), s)
        torch.cuda.synchronize()
        return rc, out.cpu(), eng.launches - n0

    n0 = eng.launches
    out = torch.empty(B, T, 2, dtype=torch.int64, device=eng.device)
    assert L.ts_pixelcnn_sample_clips(h, p(aud), p(label), None, 4, p(noise), None, None, p(out), None, B, T, None, 0, None,
                                      None, s) == 0
    torch.cuda.synchronize()
    nc = eng.launches - n0
    rc, c, n = sample(noise, None, None, None)                     # both NULL: the per-clip call, with its launches
    assert rc == 0 and torch.equal(c, out.cpu()) and n == nc
    shape = np.zeros(B, CLIP_SHAPE)
    shape[:] = (1.0, 8)
    rc, c1, n1 = sample(noise, None, shape.ctypes.data, None)      # theta 1 everywhere: the same draws, the same launches
    assert rc == 0 and torch.equal(c1, c) and n1 == nc
    assert sample(None, None, shape.ctypes.data, None)[0] == 1     # the default draw needs a noise source
    assert sample(noise, seeds, shape.ctypes.data, None)[0] == 1   # and only one
    for field, value in (("repetition_penalty", 0.5), ("repetition_penalty", float("nan")),
                         ("repetition_penalty", float("inf")), ("repetition_window", 0)):
        bad = shape.copy()
        bad[field][2] = value
        assert sample(noise, None, bad.ctypes.data, None)[0] == 1, field
        assert b"clip 2" in L.ts_last_error(h), field
    # device data the host refuses: a row of -inf still draws a code in range (the first-index argmax: 0)
    bias = torch.zeros(B, 2, 2048, device=eng.device)
    bias[1, 0] = float("-inf")
    rc, c2, _ = sample(noise, None, None, bias)
    assert rc == 0 and (c2[1, :, 0] == 0).all() and ((c2 >= 0) & (c2 < 2048)).all()
    mfcc = synth.synth_mfcc(B, 4 * T, seed=92).cuda()
    poses = torch.empty(B, 4 * T, 129, device=eng.device)
    bad = shape.copy()
    bad["repetition_window"][1] = -3
    assert L.ts_body_sample_shaped(h, p(mfcc), p(label), None, 4, p(noise), None, None, None, p(poses), B, 4 * T, None, None,
                                   bad.ctypes.data, None, s) == 1 and b"clip 1" in L.ts_last_error(h)
    assert L.ts_body_sample_shaped(h, p(mfcc), p(label), None, 4, p(noise), None, None, None, p(poses), B, 4 * T, None, None,
                                   shape.ctypes.data, p(bias), s) == 0
    torch.cuda.synchronize()


def test_two_engine_sharding(eng, ckpts):
    e2 = _engine(ckpts["pixel"], ckpts["vq"])
    try:
        B, M = 10, 48
        mfcc = synth.synth_mfcc(B, M, seed=95)
        label = torch.arange(B) % 4
        seeds = _seeds(B, 95)
        pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, 96)
        sl = lambda lo, hi: dict({k: v[lo:hi] for k, v in list(pc.items()) + list(sh.items())}, code_bias=bias[lo:hi])
        c, p = (x.cpu() for x in eng.body_generate(mfcc, label, None, seeds=seeds, code_bias=bias, **pc, **sh))
        c0, p0 = (x.cpu() for x in eng.body_generate(mfcc[:4], label[:4], None, seeds=seeds[:4], **sl(0, 4)))
        c1, p1 = (x.cpu() for x in e2.body_generate(mfcc[4:], label[4:], None, seeds=seeds[4:], **sl(4, B)))
        assert torch.equal(torch.cat([c0, c1]), c) and torch.equal(torch.cat([p0, p1]), p)
    finally:
        torch.cuda.synchronize()
        e2.close()
