"""GPU (-m gpu): sampling controls of the body prior (ts_pixelcnn_sample / ts_body_sample) on every sampler executor:
grid-wide (mode 0, forced tiles 16 / 32 / 64; mode 1, one launch per stage), cluster-resident (mode 2, 4 / 8 samples per
cluster) and the 6-D prior.

The oracle check is exact and cheap: a draw depends only on the codes before it, so one teacher-forced oracle forward over
the engine's own codes gives the logits of every draw, and the oracle's controlled draw (tests/oracle_sampling.py) on them
must reproduce each code.  By induction the whole sequence then equals the oracle's sequential generation."""
import os
import sys

import numpy as np
import pytest
import torch

import talkshow_oracle as O
from conftest import GOLDEN, ROOT
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_sampling as OS  # noqa: E402

pytestmark = pytest.mark.gpu
FIX = [(0.7, 0), (1.3, 0), (1.0, 5), (0.8, 64), (0.0, 0)]     # tests/golden/sampling.npz settings
CONFIGS = [("m0-t16", 0, {"TS_PIX_TILE": "16"}), ("m0-t32", 0, {"TS_PIX_TILE": "32"}), ("m0-t64", 0, {"TS_PIX_TILE": "64"}),
           ("m1", 1, {"TS_PIX_TILE": "64"}), ("m2-mb4", 2, {"TS_PIX3_MB": "4"}), ("m2-mb8", 2, {"TS_PIX3_MB": "8"})]


def _engine(ck, vq):
    from talkshow_b200.engine import Engine

    e = Engine(0)
    e.load_pixelcnn(ck["generator"])
    e.load_audioenc(ck["audioencoder"])
    e.load_vq(0, vq["g_body"])
    e.load_vq(1, vq["g_hand"])
    return e


@pytest.fixture(scope="module")
def eng(ckpts):
    e = _engine(ckpts["pixel"], ckpts["vq"])
    yield e
    torch.cuda.synchronize()
    e.close()


@pytest.fixture(scope="module")
def six():
    ck, vq = synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)
    e = _engine(ck, vq)
    yield e, ck, vq
    torch.cuda.synchronize()
    e.close()


@pytest.fixture
def config(request, eng, monkeypatch):
    name, mode, env = request.param
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng.set_pixelcnn_mode(mode)
    yield name
    eng.set_pixelcnn_mode(0)


_AUD = {}


def _inputs(ck, B, T, seed):
    key = (id(ck), B, T, seed)
    if key not in _AUD:
        aud = O.audio_encoder(ck["audioencoder"], synth.synth_mfcc(B, 4 * T, seed=seed))
        g = torch.Generator().manual_seed(seed + 1)
        noise = torch.empty(2 * T, B, 2048).exponential_(1, generator=g)
        _AUD[key] = (aud, torch.arange(B) % 4, noise)
    return _AUD[key]


def _sample(e, aud, label, noise, t, k, logits=False):
    out = e.pixelcnn_generate(aud, label, None if t == 0 else noise, want_logits=logits, temperature=t, top_k=k,
                              want_logp=True)
    torch.cuda.synchronize()
    return [x.cpu() for x in out]


def _check_oracle(sd, aud, label, noise, codes, t, k):
    """every code of the engine equals the oracle's controlled draw on the oracle's logits of the same prefix"""
    B, T, _ = codes.shape
    logits = O.pixelcnn_forward(sd, codes, label, aud.unsqueeze(-1).repeat(1, 1, 1, 2))       # [B,2048,T,2]
    lg = logits.permute(2, 3, 0, 1).reshape(2 * T * B, 2048)
    nz = None if t == 0 else noise.reshape(2 * T * B, 2048)
    ref = OS.draw(lg, nz, t, k).reshape(T, 2, B).permute(2, 0, 1)
    bad = (ref != codes).nonzero()
    if len(bad):
        b, i, j = bad[0].tolist()
        row = (2 * i + j) * B + b
        msg = "draw (b=%d, i=%d, j=%d): engine %d, oracle %d" % (b, i, j, codes[b, i, j], ref[b, i, j])
        if t > 0:
            keep = OS.keep_mask(lg[row], k)
            v = (torch.softmax((lg[row] / t).masked_fill(~keep, float("-inf")), -1) / nz[row]).masked_fill(~keep, -1)
            top = torch.topk(v, 2).values
            msg += "; oracle top-2 gap of p/q %.3e (rel %.3e)" % (top[0] - top[1], (top[0] - top[1]) / top[0])
        raise AssertionError("%d of %d draws differ; first %s" % (len(bad), codes.numel(), msg))


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_default_controls_bit_identical(eng, ckpts, config):
    aud, label, noise = _inputs(ckpts["pixel"], 12, 20, 11)
    ref = eng.pixelcnn_generate(aud, label, noise)
    for k in (0, 2048):
        codes, logp = _sample(eng, aud, label, noise, 1.0, k)
        assert torch.equal(codes, ref.cpu()), (config, k)
        assert torch.isfinite(logp).all() and (logp <= 0).all()


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
@pytest.mark.parametrize("B,T", [(64, 75), (12, 75), (1, 30), (100, 12)])
def test_codes_equal_oracle(eng, ckpts, config, B, T):
    if B > 16 and config.startswith("m0-t16") or B > 32 and config.startswith("m0-t32"):
        pytest.skip("tile smaller than the batch")
    aud, label, noise = _inputs(ckpts["pixel"], B, T, 100 + B)
    for t, k in FIX:
        codes, logits, logp = _sample(eng, aud, label, noise, t, k, logits=True)
        _check_oracle(ckpts["pixel"]["generator"], aud, label, noise, codes, t, k)
        # every drawn code is in the top-k set of its own logits row; logp is log_softmax of that row
        lg = logits.reshape(2 * T, B, 2048).double()
        step = codes.permute(1, 2, 0).reshape(2 * T, B)
        if k:
            kth = torch.topk(lg, k, -1).values[..., -1]
            assert (lg.gather(-1, step.unsqueeze(-1)).squeeze(-1) >= kth).all()
        ref_lp = torch.log_softmax(lg, -1).gather(-1, step.unsqueeze(-1)).squeeze(-1)
        got_lp = logp.permute(1, 2, 0).reshape(2 * T, B).double()
        assert (got_lp - ref_lp).abs().max() <= 1e-5, (t, k)


@pytest.mark.parametrize("mb", ["4", "8"])
def test_6d_codes_equal_oracle(six, monkeypatch, mb):
    e, ck, vq = six
    monkeypatch.setenv("TS_PIX3_MB", mb)
    for B, T in [(12, 10), (1, 10)]:
        aud, label, noise = _inputs(ck, B, T, 300 + B)
        ref = e.pixelcnn_generate(aud, label, noise)
        codes, _ = _sample(e, aud, label, noise, 1.0, 0)
        assert torch.equal(codes, ref.cpu())
        for t, k in FIX:
            codes, logp = _sample(e, aud, label, noise, t, k)
            _check_oracle(ck["generator"], aud, label, noise, codes, t, k)


def test_6d_full_shape(six, monkeypatch):
    """the 6-D prior at the timed shape (64 clips x 75 rows): default bit-identity for k 0 and 2048, the oracle for the
    fixture settings, greedy against the teacher-forced argmax, logp against the score, and batch independence"""
    e, ck, vq = six
    aud, label, noise = _inputs(ck, 64, 75, 364)
    ref = e.pixelcnn_generate(aud, label, noise).cpu()
    for k in (0, 2048):
        codes, _ = _sample(e, aud, label, noise, 1.0, k)
        assert torch.equal(codes, ref), k
    for t, k in FIX:
        codes, logp = _sample(e, aud, label, noise, t, k)
        _check_oracle(ck["generator"], aud, label, noise, codes, t, k)
        nll = e.pixelcnn_score(aud, label, codes).cpu()
        d = (logp + nll).abs()
        print("6-D logp vs -pixelcnn_score (%g, %d): max %.3e mean %.3e" % (t, k, d.max(), d.mean()))
        assert d.mean() <= 2.5e-5
        if t == 0:
            assert torch.equal(torch.argmax(e.pixelcnn_logits(aud, label, codes).cpu(), 1), codes)
        for b in (0, 37):
            one, lp1 = _sample(e, aud[b:b + 1], label[b:b + 1], noise[:, b:b + 1].contiguous(), t, k)
            assert torch.equal(one[0], codes[b]) and torch.equal(lp1[0], logp[b]), (t, k, b)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_tiny_temperature(eng, ckpts, six, config):
    """Any finite temperature > 0 is valid.  1e-40 (subnormal) overflows logits / t: every draw is the greedy code, every
    code lies in the codebook and logp stays finite.  1e-38 overflows only for large logits: the oracle decides."""
    for e, ck in ((eng, ckpts["pixel"]), (six[0], six[1])):
        if e is six[0] and not config.startswith("m2"):
            continue                                            # the dim 512 prior always runs on the cluster executor
        aud, label, noise = _inputs(ck, 12, 12, 71)
        greedy, _ = _sample(e, aud, label, noise, 0.0, 0)
        for k in (0, 5):
            codes, logp = _sample(e, aud, label, noise, 1e-40, k)
            assert ((codes >= 0) & (codes < 2048)).all() and torch.isfinite(logp).all()
            assert torch.equal(codes, greedy), k
            codes, logp = _sample(e, aud, label, noise, 1e-38, k)
            assert ((codes >= 0) & (codes < 2048)).all() and torch.isfinite(logp).all()
            _check_oracle(ck["generator"], aud, label, noise, codes, 1e-38, k)


def _fixture():
    return np.load(os.path.join(GOLDEN, "sampling.npz"))


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_body_sample_matches_reference_fixture(eng, six, key):
    z = _fixture()
    e = eng if key == "3d" else six[0]
    B = 3 if key == "3d" else 2
    mfcc = torch.from_numpy(z["mfcc_%s" % key]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    label = torch.full((B,), int(z["label_%s" % key]))
    for i, (t, k) in enumerate(z["settings"].tolist()):
        noise = None if t == 0 else OS.reference_noise(int(z["seed"]) + i, 2 * T, B)
        codes, poses, logp = e.body_generate(mfcc, label, noise, temperature=t, top_k=int(k), want_logp=True)
        assert torch.equal(codes.cpu(), torch.from_numpy(z["codes_%s_%d" % (key, i)])), (key, t, k)
        assert (poses.cpu()[:, ::int(z["pose_stride"])] - torch.from_numpy(z["poses_%s_%d" % (key, i)])).abs().max() <= 1e-4


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_greedy(eng, ckpts, config):
    aud, label, noise = _inputs(ckpts["pixel"], 12, 20, 21)
    g0, _ = _sample(eng, aud, label, noise, 0.0, 0)
    g1 = eng.pixelcnn_generate(aud, label, noise * 3.0 + 1.0, temperature=0.0).cpu()
    assert torch.equal(g0, g1)                                                     # noise is not read
    k1, _ = _sample(eng, aud, label, noise, 1.0, 1)
    assert torch.equal(g0, k1)                                                     # top-1 is greedy
    lg = eng.pixelcnn_logits(aud, label, g0).cpu()                                  # teacher forced [B,2048,T,2]
    assert torch.equal(torch.argmax(lg, 1), g0)


@pytest.mark.parametrize("tc", [0, 6])
def test_logp_against_score(eng, ckpts, tc):
    aud, label, noise = _inputs(ckpts["pixel"], 64, 75, 164)
    eng.set_tensor_cores(tc)
    try:
        diffs = []
        for t, k in FIX:
            codes, logp = _sample(eng, aud, label, noise, t, k)
            nll = eng.pixelcnn_score(aud, label, codes).cpu()
            diffs.append((logp + nll).abs())
        d = torch.cat([x.reshape(-1) for x in diffs])
        print("logp vs -pixelcnn_score, tensor cores %d: max %.3e mean %.3e" % (tc, d.max(), d.mean()))
        if tc == 0:
            assert d.max() <= 1e-4
        else:
            assert d.mean() <= 2.5e-5
    finally:
        eng.set_tensor_cores(6)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_batch_and_tile_independence(eng, ckpts, config):
    aud, label, noise = _inputs(ckpts["pixel"], 12, 16, 31)
    for t, k in FIX:
        full, lp = _sample(eng, aud, label, noise, t, k)
        for b in (0, 7, 11):
            one, lp1 = _sample(eng, aud[b:b + 1], label[b:b + 1], noise[:, b:b + 1].contiguous(), t, k)
            assert torch.equal(one[0], full[b]) and torch.equal(lp1[0], lp[b]), (t, k, b)


@pytest.mark.parametrize("mode", [0, 2])
def test_launch_count(eng, ckpts, mode):
    aud, label, noise = _inputs(ckpts["pixel"], 12, 20, 41)
    eng.set_pixelcnn_mode(mode)
    try:
        n0 = eng.launches
        eng.pixelcnn_generate(aud, label, noise)
        base = eng.launches - n0
        for t, k in FIX:
            n1 = eng.launches
            eng.pixelcnn_generate(aud, label, None if t == 0 else noise, temperature=t, top_k=k, want_logp=True)
            assert eng.launches - n1 == base, (t, k)
    finally:
        eng.set_pixelcnn_mode(0)


def test_error_statuses(eng, ckpts):
    import ctypes as C

    from talkshow_b200 import _lib

    aud, label, noise = _inputs(ckpts["pixel"], 2, 4, 51)
    a, lb, nz = aud.cuda(), label.cuda(), noise.cuda()
    codes = torch.empty(2, 4, 2, dtype=torch.int64, device="cuda")
    mf = synth.synth_mfcc(2, 16, seed=5).cuda()
    poses = torch.empty(2, 16, 129, device="cuda")
    s = _lib.stream_ptr(torch.device("cuda", 0))
    for t, k, n in [(-0.5, 0, nz), (float("nan"), 0, nz), (float("inf"), 0, nz), (1.0, -1, nz), (1.0, 2049, nz),
                    (0.7, 0, None)]:
        rc = eng.L.ts_pixelcnn_sample(eng.h, _lib.ptr(a), _lib.ptr(lb), _lib.ptr(n), _lib.ptr(codes), None, 2, 4, None, 0,
                                      C.c_float(t), k, None, s)
        assert rc == 1, (t, k)
        rc = eng.L.ts_body_sample(eng.h, _lib.ptr(mf), _lib.ptr(lb), _lib.ptr(n), None, _lib.ptr(poses), 2, 16,
                                  C.c_float(t), k, None, s)
        assert rc == 1, (t, k)
    assert eng.L.ts_pixelcnn_sample(eng.h, _lib.ptr(a), _lib.ptr(lb), None, _lib.ptr(codes), None, 2, 4, None, 0,
                                    C.c_float(0.0), 0, None, s) == 0
    torch.cuda.synchronize()
    for kw in [dict(temperature=-1.0), dict(top_k=4096), dict(top_k=2.5), dict(temperature=0.5, noise=None)]:
        nzk = kw.pop("noise", nz)
        with pytest.raises(ValueError):
            eng.pixelcnn_generate(a, lb, nzk, **kw)
        with pytest.raises(ValueError):
            eng.body_generate(mf, lb, nzk, **kw)


def test_wholebody_with_controls(ckpts):
    from talkshow_b200.engine import Engine
    from talkshow_b200.pipeline import WholeBody

    wb = WholeBody(Engine(0))
    wb.load(ckpts["pixel"], ckpts["vq"], ckpts["face"])
    B, M = 3, 64
    mfcc = synth.synth_mfcc(B, M, seed=61).cuda()
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(62)).cuda()
    label = torch.tensor([0, 1, 2]).cuda()
    T = M // 4
    noise = torch.empty(2 * T, B, 2048).exponential_(1, generator=torch.Generator().manual_seed(63)).cuda()
    frame = wave.shape[1] * 30 // 16000
    try:
        for t, k in FIX:
            nz = None if t == 0 else noise
            for ob in (0, 64):                         # sequential and overlapped paths
                wb.overlap_batch = ob
                out = wb.generate(mfcc, wave, label, noise=nz, temperature=t, top_k=k, keep_logp=True)
                lp = wb.last_logp
                _, body, lp2 = wb.e.body_generate(mfcc, label, nz, temperature=t, top_k=k, want_logp=True)
                face = wb.e.face_forward(wave, torch.zeros(B, 4, device="cuda"), frame)
                assert torch.equal(out, wb.e.assemble_pose(face, body)), (t, k, ob)
                assert torch.equal(lp, lp2)
            sh = wb.generate_sharded(mfcc, wave, label, 0, 1, noise_full=nz, temperature=t, top_k=k)
            assert torch.equal(sh, out)
            # world 2 on one device: rank 0 and rank 1 without the gather rebuild the single-engine result
            parts, lps = [], []
            for r in range(2):
                parts.append(wb.generate_sharded(mfcc, wave, label, r, 2, noise_full=nz, gather=False, temperature=t,
                                                 top_k=k, keep_logp=True))
                lps.append(wb.last_logp)
            assert torch.equal(torch.cat(parts), out) and torch.equal(torch.cat(lps), lp), (t, k)
    finally:
        torch.cuda.synchronize()
        wb.close()
        wb.e.close()
