"""GPU (-m gpu): nucleus (top-p) and min-p sampling of the body prior (ts_pixelcnn_sample_ctl / ts_body_sample_ctl) on every
sampler executor: grid-wide (mode 0, forced tiles 16 / 32 / 64; mode 1, one launch per stage), cluster-resident (mode 2,
4 / 8 samples per cluster) and the 6-D prior.

The keep set is built from integer sums, so codes and keep-set sizes must be equal bit for bit across executors, tiles and
batches.  One executor per shape is checked against the oracle (tests/oracle_nucleus.py) by the inductive argument of
test_gpu_sampling.py: a teacher-forced oracle forward over the engine's own codes gives the logits of every draw, and the
oracle's draw on them must reproduce each code.  The keep-set sizes are checked in float64 against the logits the engine
itself reports.  Where the CPU oracle's logits put a boundary within rounding of its threshold, the engine's draw is
checked against the oracle's draw on the engine's own logits instead."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import talkshow_oracle as O
from conftest import GOLDEN, ROOT
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_nucleus as ON  # noqa: E402
import oracle_sampling as OS  # noqa: E402

pytestmark = pytest.mark.gpu
# (temperature, top_k, top_p, min_p)
NUC = [(1.0, 0, 0.9, 0.0), (0.8, 64, 0.7, 0.0), (1.3, 0, 0.9, 0.02), (1.0, 0, 1.0, 0.05)]
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


def _configs(eng, monkeypatch, B):
    """run the body of a loop under every executor configuration that holds a batch of B"""
    for name, mode, env in CONFIGS:
        if (B > 16 and name == "m0-t16") or (B > 32 and name == "m0-t32"):
            continue
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            eng.set_pixelcnn_mode(mode)
            try:
                yield name
            finally:
                eng.set_pixelcnn_mode(0)


def _inputs(ck, B, T, seed):
    aud = O.audio_encoder(ck["audioencoder"], synth.synth_mfcc(B, 4 * T, seed=seed))
    noise = torch.empty(2 * T, B, 2048).exponential_(1, generator=torch.Generator().manual_seed(seed + 1))
    return aud, torch.arange(B) % 4, noise


def _sample(e, aud, label, noise, s, logits=False):
    t, k, p, m = s
    out = e.pixelcnn_generate(aud, label, None if t == 0 else noise, want_logits=logits, temperature=t, top_k=k, top_p=p,
                              min_p=m, want_logp=True, want_kept=True)
    torch.cuda.synchronize()
    return [x.cpu() for x in out]


def _check_oracle(sd, aud, label, noise, codes, s, own_logits):
    """Every code of the engine equals the oracle's draw on the oracle's logits of the same prefix.  The oracle's logits and
    the engine's (own_logits [2T,B,2048]) differ in their last bits, so a keep set may differ where a boundary lies within
    that rounding of its threshold: such a draw must have a boundary margin below 1e-5 and must be the oracle's draw on
    the engine's own logits, and there may be at most one in a thousand.  Any other mismatch fails with the boundary
    margins and the top-2 gap of the draw."""
    t, k, p, m = s
    B, T, _ = codes.shape
    logits = O.pixelcnn_forward(sd, codes, label, aud.unsqueeze(-1).repeat(1, 1, 1, 2))       # [B,2048,T,2]
    lg = logits.permute(2, 3, 0, 1).reshape(2 * T * B, 2048)
    nz = noise.reshape(2 * T * B, 2048)
    own = own_logits.reshape(2 * T * B, 2048)
    ref = ON.draw(lg, nz, t, k, p, m)[0].reshape(T, 2, B).permute(2, 0, 1)
    bad = (ref != codes).nonzero()
    assert len(bad) <= codes.numel() // 1000, "%d of %d draws differ" % (len(bad), codes.numel())
    for b, i, j in bad.tolist():
        row = (2 * i + j) * B + b
        keep, mp, mm = ON.keep_mask(lg[row:row + 1], t, k, p, m, return_margin=True)
        v = (torch.softmax((lg[row] / t).masked_fill(~keep[0], float("-inf")), -1) / nz[row]).masked_fill(~keep[0], -1)
        top = torch.topk(v, 2).values
        msg = ("draw (b=%d, i=%d, j=%d): engine %d, oracle %d; boundary margins top-p %.3e min-p %.3e; oracle top-2 gap of "
               "p/q rel %.3e" % (b, i, j, codes[b, i, j], ref[b, i, j], mp[0], mm[0], (top[0] - top[1]) / top[0]))
        assert min(float(mp[0]), float(mm[0])) < 1e-5, msg
        assert ON.draw(own[row:row + 1], nz[row:row + 1], t, k, p, m)[0][0] == codes[b, i, j], msg
        print("keep set within rounding of its threshold:", msg)


def _check_keep_sets(logits, codes, kept, s):
    """From the engine's own logits, in float64: every keep-set size is a valid one within rounding and holds the drawn code."""
    t, k, p, m = s
    T2, B, _ = logits.shape
    lg = logits.double()
    step = codes.permute(1, 2, 0).reshape(T2, B)
    n = kept.permute(1, 2, 0).reshape(T2, B).long()
    keep0 = OS.keep_mask(logits, k)
    tt, pp, mm = float(np.float32(t)), float(np.float32(p)), float(np.float32(m))
    z = (lg / tt)
    e = torch.exp(z - z.max(-1, keepdim=True).values).masked_fill(~keep0, 0.0)
    es, order = torch.sort(e, dim=-1, descending=True, stable=True)
    csum = torch.cumsum(es, -1)
    total = csum[..., -1]
    ls = lg.gather(-1, order)
    assert (n >= 1).all() and (n <= keep0.sum(-1)).all()
    e_code = e.gather(-1, step.unsqueeze(-1)).squeeze(-1)
    assert (e_code >= es.gather(-1, (n - 1).unsqueeze(-1)).squeeze(-1)).all(), "a drawn code lies outside its keep set"
    if m == 0 and p < 1:
        # the n most likely codes reach p, and those strictly above the boundary tie class do not
        assert (csum.gather(-1, (n - 1).unsqueeze(-1)).squeeze(-1) >= pp * (1 - 1e-5) * total).all(), s
        bound = ls.gather(-1, (n - 1).unsqueeze(-1))
        above = (es * (ls > bound)).sum(-1)
        assert (above < pp * (1 + 1e-5) * total).all(), s
        assert ((ls == bound).sum(-1) + (ls > bound).sum(-1) == n).all(), "a boundary tie class is kept whole"
    if p == 1 and m > 0:
        clear = ((e - mm).abs() > 1e-5 * mm).all(-1)
        assert clear.float().mean() > 0.9
        assert torch.equal(n[clear], (e >= mm).sum(-1)[clear]), s
    if m > 0:
        assert (e_code >= mm * (1 - 1e-5)).all()


def test_off_is_bit_identical(eng, ckpts, monkeypatch):
    """top_p = 1, min_p = 0 through the new entry point: ts_pixelcnn_sample's codes and logp, and at temperature 1 the
    default sampler's codes; the keep-set size is then the top-k count"""
    aud, label, noise = _inputs(ckpts["pixel"], 12, 20, 11)
    for name in _configs(eng, monkeypatch, 12):
        ref = eng.pixelcnn_generate(aud, label, noise).cpu()
        for t, k in [(1.0, 0), (0.7, 0), (1.0, 5), (0.0, 0)]:
            nz = None if t == 0 else noise
            old = [x.cpu() for x in eng.pixelcnn_generate(aud, label, nz, temperature=t, top_k=k, want_logp=True)]
            codes, logits, logp, kept = _sample(eng, aud, label, noise, (t, k, 1.0, 0.0), logits=True)
            assert torch.equal(codes, old[0]) and torch.equal(logp, old[1]), (name, t, k)
            if t == 1.0 and k == 0:
                assert torch.equal(codes, ref), name
            want = torch.ones_like(kept) if t == 0 else OS.keep_mask(logits, k).sum(-1).reshape(20, 2, 12).permute(2, 0, 1)
            assert torch.equal(kept.long(), want.long()), (name, t, k)


@pytest.mark.parametrize("B,T", [(64, 75), (12, 75), (1, 30), (100, 12)])
def test_codes_equal_oracle_and_every_executor(eng, ckpts, monkeypatch, B, T):
    aud, label, noise = _inputs(ckpts["pixel"], B, T, 500 + B)
    first = {}
    for name in _configs(eng, monkeypatch, B):
        for s in NUC:
            codes, logits, logp, kept = _sample(eng, aud, label, noise, s, logits=True)
            if s not in first:
                first[s] = (codes, kept, logp)
                _check_oracle(ckpts["pixel"]["generator"], aud, label, noise, codes, s, logits)
                _check_keep_sets(logits, codes, kept, s)
                lg = logits.double()
                step = codes.permute(1, 2, 0).reshape(2 * T, B)
                ref_lp = torch.log_softmax(lg, -1).gather(-1, step.unsqueeze(-1)).squeeze(-1)
                assert (logp.permute(1, 2, 0).reshape(2 * T, B).double() - ref_lp).abs().max() <= 1e-5, s
            else:
                assert torch.equal(codes, first[s][0]) and torch.equal(kept, first[s][1]), (name, s)
                assert torch.equal(logp, first[s][2]), (name, s)
    if B == 64:                                                   # a sample alone and in batches of 12 and 64
        for s in NUC:
            for b in (0, 5, 11):
                for nb in (1, 12):
                    sl = slice(b, b + 1) if nb == 1 else slice(0, 12)
                    c, lp, kp = _sample(eng, aud[sl], label[sl], noise[:, sl].contiguous(), s)
                    at = 0 if nb == 1 else b
                    assert torch.equal(c[at], first[s][0][b]) and torch.equal(kp[at], first[s][1][b]), (s, b, nb)


@pytest.mark.parametrize("mb", ["4", "8"])
def test_6d_prior(six, monkeypatch, mb):
    e, ck, vq = six
    monkeypatch.setenv("TS_PIX3_MB", mb)
    for B, T in [(12, 10), (1, 10)]:
        aud, label, noise = _inputs(ck, B, T, 700 + B)
        ref = e.pixelcnn_generate(aud, label, noise).cpu()
        assert torch.equal(_sample(e, aud, label, noise, (1.0, 0, 1.0, 0.0))[0], ref)
        for s in NUC:
            codes, logits, logp, kept = _sample(e, aud, label, noise, s, logits=True)
            _check_oracle(ck["generator"], aud, label, noise, codes, s, logits)
            _check_keep_sets(logits, codes, kept, s)


def test_tiny_top_p_is_greedy(eng, ckpts, monkeypatch):
    aud, label, noise = _inputs(ckpts["pixel"], 12, 20, 21)
    for name in _configs(eng, monkeypatch, 12):
        codes, logits, _, kept = _sample(eng, aud, label, noise, (1.0, 0, 1e-6, 0.0), logits=True)
        greedy = eng.pixelcnn_generate(aud, label, None, temperature=0.0).cpu()
        ties = (logits == logits.max(-1, keepdim=True).values).sum(-1).reshape(20, 2, 12).permute(2, 0, 1)
        assert (ties == 1).all(), "the inputs were chosen without tied maxima"
        assert torch.equal(codes, greedy) and torch.equal(kept.long(), ties), name
        one = _sample(eng, aud, label, noise, (0.9, 0, 1.0, 1.0))                          # min_p = 1: the ties of the maximum
        assert torch.equal(one[0], greedy) and (one[2] == 1).all(), name


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_body_sample_matches_reference_fixture(eng, six, key):
    z = np.load(os.path.join(GOLDEN, "sampling_p.npz"))
    e = eng if key == "3d" else six[0]
    B = 3 if key == "3d" else 2
    mfcc = torch.from_numpy(z["mfcc_%s" % key]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    label = torch.full((B,), int(z["label_%s" % key]))
    for i, (t, k, p, m) in enumerate(z["settings"].tolist()):
        noise = OS.reference_noise(int(z["seeds_%s" % key][i]), 2 * T, B)
        codes, poses, kept = e.body_generate(mfcc, label, noise, temperature=t, top_k=int(k), top_p=p, min_p=m, want_kept=True)
        assert torch.equal(codes.cpu(), torch.from_numpy(z["codes_%s_%d" % (key, i)])), (key, t, k, p, m)
        assert (poses.cpu()[:, ::int(z["pose_stride"])] - torch.from_numpy(z["poses_%s_%d" % (key, i)])).abs().max() <= 1e-4
        # the engine's logits differ from the CPU's in the last bits: a keep set may differ where the fixture's margin is
        # of that order, the codes may not
        same = (kept.cpu() == torch.from_numpy(z["kept_%s_%d" % (key, i)])).float().mean()
        print("fixture %s %s: %.4f of the keep-set sizes equal the CPU's" % (key, (t, k, p, m), same))
        assert same >= 0.98


@pytest.mark.parametrize("mode", [0, 2])
def test_launch_count(eng, ckpts, mode):
    aud, label, noise = _inputs(ckpts["pixel"], 12, 20, 41)
    eng.set_pixelcnn_mode(mode)
    try:
        n0 = eng.launches
        eng.pixelcnn_generate(aud, label, noise)
        base = eng.launches - n0
        for t, k, p, m in NUC:
            n1 = eng.launches
            eng.pixelcnn_generate(aud, label, noise, temperature=t, top_k=k, top_p=p, min_p=m, want_logp=True, want_kept=True)
            assert eng.launches - n1 == base, (t, k, p, m)
    finally:
        eng.set_pixelcnn_mode(0)


def test_error_statuses(eng, ckpts):
    from talkshow_b200 import _lib

    aud, label, noise = _inputs(ckpts["pixel"], 2, 4, 51)
    a, lb, nz = aud.cuda(), label.cuda(), noise.cuda()
    codes = torch.empty(2, 4, 2, dtype=torch.int64, device="cuda")
    mf = synth.synth_mfcc(2, 16, seed=5).cuda()
    poses = torch.empty(2, 16, 129, device="cuda")
    s = _lib.stream_ptr(torch.device("cuda", 0))

    def both(ctl, n=nz):
        ref = None if ctl is None else C.byref(ctl)
        return (eng.L.ts_pixelcnn_sample_ctl(eng.h, _lib.ptr(a), _lib.ptr(lb), _lib.ptr(n), _lib.ptr(codes), None, 2, 4, None, 0, ref, s),
                eng.L.ts_body_sample_ctl(eng.h, _lib.ptr(mf), _lib.ptr(lb), _lib.ptr(n), None, _lib.ptr(poses), 2, 16, ref, s))

    mk = lambda t=1.0, k=0, p=1.0, m=0.0: _lib.ts_sample_ctl(t, k, p, m, None, None)
    for bad in [mk(p=0.0), mk(p=-0.5), mk(p=1.5), mk(p=float("nan")), mk(m=-0.1), mk(m=1.5), mk(m=float("nan")), mk(t=-1.0),
                mk(k=2049), mk(t=float("inf"))]:
        assert both(bad) == (1, 1), (bad.temperature, bad.top_k, bad.top_p, bad.min_p)
    assert both(None) == (1, 1)
    assert both(mk(t=0.7, p=0.9), None) == (1, 1)                                    # sampling without noise
    assert both(mk(t=0.0, p=0.9), None) == (0, 0)                                    # greedy needs none
    assert both(mk(p=0.9, m=1.0)) == (0, 0)
    torch.cuda.synchronize()
    # the entry points without the struct are unchanged
    assert eng.L.ts_pixelcnn_sample(eng.h, _lib.ptr(a), _lib.ptr(lb), _lib.ptr(nz), _lib.ptr(codes), None, 2, 4, None, 0,
                                    C.c_float(1.0), 2049, None, s) == 1
    assert eng.L.ts_body_sample(eng.h, _lib.ptr(mf), _lib.ptr(lb), None, None, _lib.ptr(poses), 2, 16, C.c_float(0.5), 0, None, s) == 1
    assert eng.L.ts_pixelcnn_sample(eng.h, _lib.ptr(a), _lib.ptr(lb), None, _lib.ptr(codes), None, 2, 4, None, 0,
                                    C.c_float(0.0), 0, None, s) == 0
    torch.cuda.synchronize()
    for kw in [dict(top_p=0.0), dict(top_p=1.1), dict(min_p=-0.5), dict(min_p=2.0)]:
        with pytest.raises(ValueError):
            eng.pixelcnn_generate(a, lb, nz, **kw)
        with pytest.raises(ValueError):
            eng.body_generate(mf, lb, nz, **kw)


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
        for t, k, p, m in NUC:
            ctl = dict(temperature=t, top_k=k, top_p=p, min_p=m)
            for ob in (0, 64):                         # sequential and overlapped paths
                wb.overlap_batch = ob
                out = wb.generate(mfcc, wave, label, noise=noise, keep_logp=True, **ctl)
                lp, kp = wb.last_logp, wb.last_kept
                _, body, lp2, kp2 = wb.e.body_generate(mfcc, label, noise, want_logp=True, want_kept=True, **ctl)
                face = wb.e.face_forward(wave, torch.zeros(B, 4, device="cuda"), frame)
                assert torch.equal(out, wb.e.assemble_pose(face, body)), (ctl, ob)
                assert torch.equal(lp, lp2) and torch.equal(kp, kp2)
            assert torch.equal(wb.generate_sharded(mfcc, wave, label, 0, 1, noise_full=noise, **ctl), out)
            parts, lps, kps = [], [], []
            for r in range(2):                         # world 2 on one device, without the gather
                parts.append(wb.generate_sharded(mfcc, wave, label, r, 2, noise_full=noise, gather=False, keep_logp=True, **ctl))
                lps.append(wb.last_logp)
                kps.append(wb.last_kept)
            assert torch.equal(torch.cat(parts), out) and torch.equal(torch.cat(lps), lp) and torch.equal(torch.cat(kps), kp), ctl
    finally:
        torch.cuda.synchronize()
        wb.close()
        wb.e.close()
