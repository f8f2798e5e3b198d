"""GPU (-m gpu): styled sampling of the body prior (ts_pixelcnn_sample_styled, ts_body_sample_styled,
ts_pixelcnn_score_styled) on every sampler executor of test_gpu_seeded.CONFIGS and on the 6-D prior, with explicit noise
and with seeds.

Pinned bit for bit: a one-hot schedule is the labelled call; the reference fixture's codes (tests/golden/style.npz); the
rows before a switch are those of the constant schedule; every executor gives the same bits; a clip gives the same bits
alone and in a batch of other schedules.  Per-row schedules are checked against the oracle's draw on its full-grid
teacher-forced logits of the engine's own codes (tests/oracle_style.py), and the row each gate reads is checked by the
teacher-forced scorer: the sampler's log p of every draw equals -nll of pixelcnn_score(style=) on the same codes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from talkshow_b200 import _lib, synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_sampling as OSM  # noqa: E402
import oracle_style as OST  # noqa: E402
from test_gpu_seeded import CONFIGS, SETTINGS, _aud, _engine, _seeds, _wrapper, config, eng, six  # noqa: E402,F401

pytestmark = pytest.mark.gpu
SOURCES = ("noise", "seeds")
SHAPES = [(64, 75), (12, 75), (1, 30), (100, 12)]
# sampler log p against -nll of the scorer on the same codes: the scorer's dense layers run on the split-operand wgmma
# kernel, which puts the unstyled pair 4.6e-5 apart at 64 x 75 (DESIGN §8).  A gate that read a neighbouring row's style
# moves its class term by the difference of two embedding rows, orders of magnitude more.
LOGP_SCORE_TOL = 5e-5


def _run(e, aud, label, s, src, seeds, noise, **kw):
    """[codes, logp, kept] of one call (None where the call has none); s None: the default draw"""
    greedy = s is not None and s["temperature"] == 0
    n = None if greedy or src != "noise" else noise
    sd = None if greedy or src != "seeds" else seeds
    if s is None:
        return [e.pixelcnn_generate(aud, label, n, seeds=sd, **kw).cpu(), None, None]
    want_kept = "top_p" in s
    out = [x.cpu() for x in e.pixelcnn_generate(aud, label, n, seeds=sd, want_logp=True, want_kept=want_kept, **s, **kw)]
    return [out[0], out[1], out[2] if want_kept else None]


def _equal(a, b, what, logp_tol=0.0):
    for x, y, n in zip(a, b, ("codes", "logp", "kept")):
        if x is not None or y is not None:
            assert x is not None and y is not None and x.shape == y.shape, (what, n)
            if n == "logp" and logp_tol:
                assert (x - y).abs().max() <= logp_tol, (what, n)
            else:
                bad = x != y
                assert not bad.any(), (what, n, int(bad.sum()), bad.nonzero()[:4].tolist())


def _tol(config):
    """log p tolerance between two calls: the cluster executor has been seen to give log p values of two calls that must
    agree differing in the last bits with every code equal (the open issue of DESIGN §3d, also without styles), so its
    log p is compared at 1e-5; everything else bit for bit"""
    return 1e-5 if config.startswith("m2") else 0.0


def _skip_tile(config, B):
    if B > 16 and config.startswith("m0-t16") or B > 32 and config.startswith("m0-t32"):
        pytest.skip("tile smaller than the batch")


def _onehot(label, H):
    return OST.onehot(label, 4, H)


def _schedules(B, H, seed):
    """per-row schedules [B,H,4]: a step switch at H // 2, a linear fade over the middle half, random convex rows"""
    a, b = torch.arange(B) % 4, (torch.arange(B) + 1) % 4
    step = _onehot(a, H).clone()
    step[:, H // 2:] = _onehot(b, H - H // 2)
    r0, r1 = H // 4, max(H // 4 + 1, 3 * H // 4)
    t = ((torch.arange(H, dtype=torch.float64) - r0) / (r1 - r0)).clamp(0, 1)
    fade = (1 - t)[None, :, None] * _onehot(a, H).double() + t[None, :, None] * _onehot((a + 2) % 4, H).double()
    w = torch.rand(B, H, 4, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) ** 2
    rand = w / w.sum(-1, keepdim=True)
    return {"step": step, "fade": fade.float(), "random": rand.float()}


def _oracle_codes(sd, aud, style, codes, noise):
    """the oracle's default draw of every position on its full-grid teacher-forced logits of ``codes`` under ``style``"""
    B, T = codes.shape[:2]
    logits = OST.pixelcnn_forward(sd, codes, style, aud.unsqueeze(-1).repeat(1, 1, 1, 2))          # [B,2048,T,2]
    lg = logits.permute(2, 3, 0, 1).reshape(2 * T * B, 2048)
    return OSM.draw(lg, noise.reshape(2 * T * B, 2048), 1.0, 0).reshape(T, 2, B).permute(2, 0, 1)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
@pytest.mark.parametrize("B,T", SHAPES)
def test_onehot_equals_label(eng, ckpts, config, B, T):
    """a one-hot schedule of each clip's class is the labelled call, with the launches of the anchored call"""
    _skip_tile(config, B)
    aud, label = _aud(ckpts["pixel"], B, T, 100 + B)
    seeds = _seeds(B, B + T)
    noise = eng.sampler_noise(seeds, T)
    free = torch.full((B, T, 2), -1, dtype=torch.int64)
    for src in SOURCES:
        for s in SETTINGS:
            ref = _run(eng, aud, label, s, src, seeds, noise)
            n0 = eng.launches
            _run(eng, aud, label, s, src, seeds, noise, anchors=free)
            n1 = eng.launches
            got = _run(eng, aud, None, s, src, seeds, noise, style=_onehot(label, T))
            assert eng.launches - n1 == n1 - n0, (config, s, src)
            _equal(got, ref, (config, B, T, s, src), _tol(config))


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_onehot_with_anchors_prefix_and_every_class(eng, ckpts, config):
    B, T, T0 = 12, 20, 6
    aud, _ = _aud(ckpts["pixel"], B, T0 + T, 41)
    seeds = _seeds(B, 41)
    pre = torch.randint(0, 2048, (B, T0, 2), generator=torch.Generator().manual_seed(42))
    anchors = torch.where(torch.rand(B, T, 2, generator=torch.Generator().manual_seed(43)) < 0.3,
                          torch.randint(0, 2048, (B, T, 2), generator=torch.Generator().manual_seed(44)), -1)
    for cls in range(4):
        label = torch.full((B,), cls, dtype=torch.int64)
        for s in (None, SETTINGS[1], SETTINGS[-1]):
            kw = dict(T=T, pre_latents=pre, anchors=anchors)
            ref = _run(eng, aud, label, s, "seeds", seeds, None, **kw)
            got = _run(eng, aud, None, s, "seeds", seeds, None, style=_onehot(label, T0 + T), **kw)
            _equal(got, ref, (config, cls, s), _tol(config))


def test_onehot_body_generate(eng, ckpts):
    B, M = 6, 64
    mfcc = synth.synth_mfcc(B, M, seed=51)
    label = torch.tensor([0, 1, 2, 3, 1, 2])
    seeds = _seeds(B, 51)
    for s in (dict(), dict(temperature=0.8, top_k=50, want_logp=True), dict(top_p=0.9, want_logp=True, want_kept=True)):
        ref = [x.cpu() for x in eng.body_generate(mfcc, label, None, seeds=seeds, **s)]
        got = [x.cpu() for x in eng.body_generate(mfcc, None, None, seeds=seeds, style=_onehot(label, M // 4), **s)]
        for x, y in zip(got, ref):
            assert torch.equal(x, y), s


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_reference_fixture(eng, six, geo):
    z = np.load(os.path.join(GOLDEN, "style.npz"))
    z = {k[3:]: z[k] for k in z.files if k.startswith(geo + "_")}
    e = eng if geo == "3d" else six[0]
    audio = torch.from_numpy(z["audio"])
    B, T = z["codes"].shape[1:3]
    for i, name in enumerate(str(n) for n in z["cases"]):
        noise = OSM.reference_noise(int(z["seed"][i]), 2 * T, B)
        w = torch.from_numpy(z["weights"][i])
        codes = e.pixelcnn_generate(audio, None, noise, style=w).cpu()
        assert torch.equal(codes, torch.from_numpy(z["codes"][i])), (geo, name)
        if geo == "3d":
            g = _wrapper(e)
            g.generate(torch.from_numpy(z["mfcc"]), torch.tensor([0]), noise_fn=lambda T_, B_: noise, style=w)
            assert torch.equal(g.last_codes.cpu(), torch.from_numpy(z["codes"][i])), (geo, name)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
@pytest.mark.parametrize("B,T", SHAPES)
def test_schedules_match_oracle_and_scorer(eng, ckpts, config, B, T):
    """per-row schedules: the codes are the oracle's draw on its own teacher-forced logits of them; every draw's log p
    equals -nll of the styled scorer on the same codes; the scorer's logits equal the oracle's full-grid forward"""
    _skip_tile(config, B)
    aud, _ = _aud(ckpts["pixel"], B, T, 200 + B)
    seeds = _seeds(B, 7 * B + T)
    noise = eng.sampler_noise(seeds, T).cpu()
    for kind, st in _schedules(B, T, B + T).items():
        codes, logp = (x.cpu() for x in eng.pixelcnn_generate(aud, None, None, seeds=seeds, style=st, want_logp=True))
        assert torch.equal(codes, _oracle_codes(ckpts["pixel"]["generator"], aud, st, codes, noise)), (config, kind)
        nll, logits = eng.pixelcnn_score(aud, None, codes, want_logits=True, style=st)
        assert (logp + nll.cpu()).abs().max() <= LOGP_SCORE_TOL, (config, kind)
        if config == "m0-t64" or B == 1:
            _, ref = OST.score(ckpts["pixel"]["generator"], aud, st, codes)
            assert (logits.cpu() - ref).abs().max() <= 1e-4, (config, kind)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_switch_prefix_identity(eng, ckpts, config):
    B, T, k = 12, 40, 17
    aud, _ = _aud(ckpts["pixel"], B, T, 61)
    seeds = _seeds(B, 61)
    noise = eng.sampler_noise(seeds, T)
    a = torch.tensor([0.5, 0.0, 0.5, 0.0]).expand(B, T, 4).contiguous()
    sw = a.clone()
    sw[:, k:] = torch.tensor([0.0, 0.25, 0.0, 0.75])
    for src in SOURCES:
        for s in SETTINGS:
            ref = _run(eng, aud, None, s, src, seeds, noise, style=a)
            got = _run(eng, aud, None, s, src, seeds, noise, style=sw)
            _equal([x if x is None else x[:, :k] for x in got], [x if x is None else x[:, :k] for x in ref], (config, s, src),
                   _tol(config))


def test_executors_bit_identical(eng, ckpts, monkeypatch):
    B, T = 12, 30
    aud, _ = _aud(ckpts["pixel"], B, T, 71)
    seeds = _seeds(B, 71)
    st = _schedules(B, T, 72)["random"]
    ref = {}
    for name, mode, env in CONFIGS:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng.set_pixelcnn_mode(mode)
        for i, s in enumerate(SETTINGS):
            got = _run(eng, aud, None, s, "seeds", seeds, None, style=st)
            if i in ref:
                _equal(got, ref[i], (name, s), _tol(name))
            else:
                ref[i] = got
        for k in env:
            monkeypatch.delenv(k)
    eng.set_pixelcnn_mode(0)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_clip_alone_equals_clip_in_batch(eng, ckpts, config):
    B, T = 12, 16
    aud, _ = _aud(ckpts["pixel"], B, T, 81)
    seeds = _seeds(B, 81)
    st = _schedules(B, T, 82)["random"]
    for s in (None, SETTINGS[2], SETTINGS[-1]):
        full = _run(eng, aud, None, s, "seeds", seeds, None, style=st)
        for b in (0, 7, 11):
            one = _run(eng, aud[b:b + 1], None, s, "seeds", seeds[b:b + 1], None, style=st[b:b + 1])
            _equal(one, [x if x is None else x[b:b + 1] for x in full], (config, s, b), _tol(config))


def test_null_style_and_error_statuses(eng, ckpts):
    """style = NULL equals the anchored and score entry points with their launches; bad class inputs are refused"""
    B, T = 4, 12
    aud, label = _aud(ckpts["pixel"], B, T, 91)
    aud = aud.cuda().contiguous()
    label = label.cuda()
    noise = eng.sampler_noise(_seeds(B, 91), T)
    st = _onehot(label.cpu(), T).cuda()
    L, h, p = eng.L, eng.h, _lib.ptr
    s = _lib.stream_ptr(eng.device)

    def sample(fn, *head):
        out = torch.empty(B, T, 2, dtype=torch.int64, device=eng.device)
        n0 = eng.launches
        rc = fn(h, p(aud), *head, p(noise), None, None, p(out), None, B, T, None, 0, None, s)
        torch.cuda.synchronize()
        return rc, out.cpu(), eng.launches - n0

    rc0, c0, n0 = sample(L.ts_pixelcnn_sample_anchored, p(label))
    rc1, c1, n1 = sample(L.ts_pixelcnn_sample_styled, p(label), None, 4)
    assert rc0 == rc1 == 0 and torch.equal(c0, c1) and n0 == n1
    rc2, c2, n2 = sample(L.ts_pixelcnn_sample_styled, None, p(st), 4)
    assert rc2 == 0 and torch.equal(c2, c0) and n2 == n0
    for lab, sty, ncls in ((None, None, 4), (p(label), p(st), 3), (None, p(st), 5), (None, p(st), 17), (None, p(st), 0)):
        rc, _, _ = sample(L.ts_pixelcnn_sample_styled, lab, sty, ncls)
        assert rc == 1, (lab, ncls)
    codes = c0.cuda()
    mfcc = synth.synth_mfcc(B, 4 * T, seed=92).cuda()
    poses = torch.empty(B, 4 * T, 129, device=eng.device)
    assert L.ts_body_sample_styled(h, p(mfcc), None, p(st), 3, p(noise), None, None, None, p(poses), B, 4 * T, None, s) == 1
    nll0, nll1 = (torch.empty(B, T, 2, device=eng.device) for _ in range(2))
    n0 = eng.launches
    assert L.ts_pixelcnn_score(h, p(aud), p(label), p(codes), p(nll0), None, B, T, s) == 0
    n1 = eng.launches
    assert L.ts_pixelcnn_score_styled(h, p(aud), p(label), None, 4, p(codes), p(nll1), None, B, T, s) == 0
    assert eng.launches - n1 == n1 - n0
    assert torch.equal(nll0, nll1)
    assert L.ts_pixelcnn_score_styled(h, p(aud), None, p(st), 4, p(codes), p(nll1), None, B, T, s) == 0
    assert torch.equal(nll0, nll1)
    assert L.ts_pixelcnn_score_styled(h, p(aud), None, p(st), 2, p(codes), p(nll1), None, B, T, s) == 1
    assert L.ts_pixelcnn_score_styled(h, p(aud), None, None, 4, p(codes), p(nll1), None, B, T, s) == 1


def test_two_engine_sharding(eng, ckpts):
    e2 = _engine(ckpts["pixel"], ckpts["vq"])
    try:
        B, M = 10, 48
        mfcc = synth.synth_mfcc(B, M, seed=95)
        seeds = _seeds(B, 95)
        st = _schedules(B, M // 4, 96)["fade"]
        c, p = (x.cpu() for x in eng.body_generate(mfcc, None, None, seeds=seeds, style=st))
        c0, p0 = (x.cpu() for x in eng.body_generate(mfcc[:4], None, None, seeds=seeds[:4], style=st[:4]))
        c1, p1 = (x.cpu() for x in e2.body_generate(mfcc[4:], None, None, seeds=seeds[4:], style=st[4:]))
        assert torch.equal(torch.cat([c0, c1]), c) and torch.equal(torch.cat([p0, p1]), p)
    finally:
        torch.cuda.synchronize()
        e2.close()


def test_6d(six, monkeypatch):
    """the 6-D prior on the cluster executor: one-hot equals the label, schedules match the oracle and the scorer.  log p
    of separate calls is compared at 1e-5 (the open last-bit issue of DESIGN §3d), codes bit for bit."""
    e, ck, _ = six
    for mb in ("4", "8"):
        monkeypatch.setenv("TS_PIX3_MB", mb)
        for B, T in [(64, 10), (12, 10), (1, 10)]:
            aud, label = _aud(ck, B, T, 300 + B)
            seeds = _seeds(B, B)
            noise = e.sampler_noise(seeds, T)
            for src in SOURCES:
                for s in SETTINGS:
                    ref = _run(e, aud, label, s, src, seeds, noise)
                    got = _run(e, aud, None, s, src, seeds, noise, style=_onehot(label, T))
                    _equal(got, ref, (mb, B, T, s, src), logp_tol=1e-5)
            for kind, st in _schedules(B, T, 7 * B).items():
                codes, logp = (x.cpu() for x in e.pixelcnn_generate(aud, None, None, seeds=seeds, style=st, want_logp=True))
                assert torch.equal(codes, _oracle_codes(ck["generator"], aud, st, codes, noise.cpu())), (mb, B, kind)
                nll = e.pixelcnn_score(aud, None, codes, style=st).cpu()
                assert (logp + nll).abs().max() <= LOGP_SCORE_TOL, (mb, B, kind)
