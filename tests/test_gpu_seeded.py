"""GPU (-m gpu): seeded sampling of the body prior (ts_sampler_noise, ts_pixelcnn_sample_seeded, ts_body_sample_seeded) on
every sampler executor: grid-wide (mode 0 with forced tiles 16 / 32 / 64; mode 1, one launch per stage), cluster-resident
(mode 2 with 4 / 8 samples per cluster) and the 6-D prior.

The stated equivalence is the backbone: a seeded call equals, bit for bit, the explicit-noise call fed with the noise
ts_sampler_noise materialises, and that noise equals the numpy RNG contract (tests/oracle_seeded.py) to one ulp of -log.
The oracle check then is the one of test_gpu_sampling.py: the oracle's draw on its teacher-forced logits of the engine's
own codes, with the materialised noise, reproduces every code."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

import talkshow_oracle as O
from conftest import GOLDEN, ROOT
from talkshow_b200 import _lib, synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_sampling as OSM  # noqa: E402
import oracle_seeded as OS  # noqa: E402

pytestmark = pytest.mark.gpu
CONFIGS = [("m0-t16", 0, {"TS_PIX_TILE": "16"}), ("m0-t32", 0, {"TS_PIX_TILE": "32"}), ("m0-t64", 0, {"TS_PIX_TILE": "64"}),
           ("m1", 1, {"TS_PIX_TILE": "64"}), ("m2-mb4", 2, {"TS_PIX3_MB": "4"}), ("m2-mb8", 2, {"TS_PIX3_MB": "8"})]


def _settings():
    """None (the default draw), then the control settings of tests/golden/sampling.npz and sampling_p.npz"""
    s = [None]
    s += [dict(temperature=float(t), top_k=int(k)) for t, k in np.load(os.path.join(GOLDEN, "sampling.npz"))["settings"].tolist()]
    s += [dict(temperature=float(t), top_k=int(k), top_p=float(p), min_p=float(m))
          for t, k, p, m in np.load(os.path.join(GOLDEN, "sampling_p.npz"))["settings"].tolist()]
    return s


SETTINGS = _settings()


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


def _aud(ck, B, T, seed):
    key = (id(ck), B, T, seed)
    if key not in _AUD:
        _AUD[key] = (O.audio_encoder(ck["audioencoder"], synth.synth_mfcc(B, 4 * T, seed=seed)), torch.arange(B) % 4)
    return _AUD[key]


def _seeds(B, base):
    return torch.tensor([base * 1000003 + 7919 * b - (b % 3) * 2 ** 40 for b in range(B)], dtype=torch.int64)


def _run(e, aud, label, s, noise=None, seeds=None, **kw):
    """codes, logp, kept (None where the setting has none) of one call with explicit noise or seeds"""
    if s is None:
        return [e.pixelcnn_generate(aud, label, noise, seeds=seeds, **kw).cpu(), None, None]
    want_kept = "top_p" in s
    greedy = s["temperature"] == 0
    out = e.pixelcnn_generate(aud, label, None if greedy else noise, seeds=None if greedy else seeds, want_logp=True,
                              want_kept=want_kept, **s, **kw)
    out = [x.cpu() for x in out]
    return out + [None] * (3 - len(out))


def _equal(a, b, what):
    for x, y, n in zip(a, b, ("codes", "logp", "kept")):
        if x is not None or y is not None:
            assert torch.equal(x, y), (what, n)


def test_sampler_noise_matches_numpy_contract(eng):
    for B, T, T0 in [(3, 5, 0), (2, 4, 7), (1, 1, 0), (65, 2, 3)]:
        seeds = _seeds(B, T + T0)
        seeds[0] = -1 if B > 1 else seeds[0]
        got = eng.sampler_noise(seeds, T, T0).cpu().numpy()
        ref = OS.noise(seeds.tolist(), T, T0)
        assert got.shape == (2 * T, B, 2048)
        ulp = np.abs(np.nextafter(ref, np.float32(np.inf)) - ref)
        assert (np.abs(got - ref) <= ulp).all(), (B, T, T0, np.abs(got - ref).max())
        assert (got > 0).all() and np.isfinite(got).all()
    # a T0 call is the tail of a longer one, a clip's block is its own
    s = _seeds(4, 1)
    full = eng.sampler_noise(s, 6).cpu()
    assert torch.equal(eng.sampler_noise(s, 2, 4).cpu(), full[8:])
    assert torch.equal(eng.sampler_noise(s[2:3], 6).cpu()[:, 0], full[:, 2])


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
@pytest.mark.parametrize("B,T", [(64, 75), (12, 75), (1, 30), (100, 12)])
def test_seeded_equals_explicit(eng, ckpts, config, B, T):
    if B > 16 and config.startswith("m0-t16") or B > 32 and config.startswith("m0-t32"):
        pytest.skip("tile smaller than the batch")
    aud, label = _aud(ckpts["pixel"], B, T, 100 + B)
    seeds = _seeds(B, B + T)
    noise = eng.sampler_noise(seeds, T)
    for s in SETTINGS:
        _equal(_run(eng, aud, label, s, seeds=seeds), _run(eng, aud, label, s, noise=noise), (config, B, T, s))


def test_seeded_equals_explicit_6d(six, monkeypatch):
    e, ck, _ = six
    for mb in ("4", "8"):
        monkeypatch.setenv("TS_PIX3_MB", mb)
        for B, T in [(64, 10), (12, 10), (1, 10)]:
            aud, label = _aud(ck, B, T, 300 + B)
            seeds = _seeds(B, B)
            noise = e.sampler_noise(seeds, T)
            for s in SETTINGS:
                _equal(_run(e, aud, label, s, seeds=seeds), _run(e, aud, label, s, noise=noise), (mb, B, T, s))


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_codes_equal_oracle(eng, six, ckpts, geo):
    e, ck = (eng, ckpts["pixel"]) if geo == "3d" else (six[0], six[1])
    B, T = (12, 75) if geo == "3d" else (12, 10)
    aud, label = _aud(ck, B, T, 500)
    seeds = _seeds(B, 5)
    codes = e.pixelcnn_generate(aud, label, None, seeds=seeds).cpu()
    noise = torch.from_numpy(OS.noise(seeds.tolist(), T))
    logits = O.pixelcnn_forward(ck["generator"], codes, label, aud.unsqueeze(-1).repeat(1, 1, 1, 2))     # [B,2048,T,2]
    lg = logits.permute(2, 3, 0, 1).reshape(2 * T * B, 2048)
    ref = OSM.draw(lg, noise.reshape(2 * T * B, 2048), 1.0, 0).reshape(T, 2, B).permute(2, 0, 1)
    assert torch.equal(ref, codes), int((ref != codes).sum())


def _batch_invariance(e, aud, label, settings):
    s = 424242
    seeds = _seeds(12, 9)
    for b in (0, 7, 11):
        seeds[b] = s
    for st in settings:
        full = _run(e, aud, label, st, seeds=seeds)
        for b in (0, 7, 11):
            one = _run(e, aud[b:b + 1], label[b:b + 1], st, seeds=torch.tensor([s]))
            assert torch.equal(one[0][0], full[0][b]), (st, b)
            if st is not None:
                assert torch.equal(one[1][0], full[1][b]), (st, b)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_batch_invariance(eng, ckpts, config):
    aud, label = _aud(ckpts["pixel"], 12, 16, 31)
    _batch_invariance(eng, aud, label, SETTINGS[:3] + SETTINGS[-2:])


def test_batch_invariance_6d(six):
    e, ck, _ = six
    aud, label = _aud(ck, 12, 10, 33)
    _batch_invariance(e, aud, label, SETTINGS[:3] + SETTINGS[-2:])


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_body_generate_batch_invariance(eng, six, geo):
    e = eng if geo == "3d" else six[0]
    B, M = 12, 64
    mfcc = synth.synth_mfcc(B, M, seed=71).cuda()
    label = (torch.arange(B) % 4).cuda()
    seeds = _seeds(B, 3)
    codes, poses = e.body_generate(mfcc, label, None, seeds=seeds)
    for b in (0, 7, 11):
        c1, p1 = e.body_generate(mfcc[b:b + 1], label[b:b + 1], None, seeds=seeds[b:b + 1])
        assert torch.equal(c1[0], codes[b])
        assert torch.equal(p1[0], poses[b]), (b, (p1[0] - poses[b]).abs().max().item())
    # and the seeded body call equals the explicit one on the materialised noise
    c2, p2 = e.body_generate(mfcc, label, e.sampler_noise(seeds, M // 4))
    assert torch.equal(c2, codes) and torch.equal(p2, poses)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_prefix_rows_keyed_from_T0(eng, ckpts, config):
    B, T0, T = 5, 6, 10
    aud, label = _aud(ckpts["pixel"], B, T0 + T, 41)
    pre = torch.randint(0, 2048, (B, T0, 2), generator=torch.Generator().manual_seed(42))
    seeds = _seeds(B, 4)
    noise = eng.sampler_noise(seeds, T, T0)
    for s in (None, SETTINGS[1], SETTINGS[-2]):
        got = _run(eng, aud, label, s, seeds=seeds, T=T, pre_latents=pre)
        _equal(got, _run(eng, aud, label, s, noise=noise, T=T, pre_latents=pre), (config, s))
    # not the noise of rows 0..T-1
    other = _run(eng, aud, label, None, noise=eng.sampler_noise(seeds, T), T=T, pre_latents=pre)
    assert not torch.equal(other[0], _run(eng, aud, label, None, seeds=seeds, T=T, pre_latents=pre)[0])


@pytest.mark.parametrize("mode", [0, 2])
def test_launch_counts(eng, ckpts, mode):
    aud, label = _aud(ckpts["pixel"], 12, 20, 43)
    seeds = _seeds(12, 1)
    noise = eng.sampler_noise(seeds, 20)
    mfcc = synth.synth_mfcc(12, 80, seed=44).cuda()
    eng.set_pixelcnn_mode(mode)
    try:
        n0 = eng.launches
        eng.pixelcnn_generate(aud, label, noise)
        base = eng.launches - n0
        for s in SETTINGS:
            n1 = eng.launches
            _run(eng, aud, label, s, seeds=seeds)
            assert eng.launches - n1 == base, s
        n0 = eng.launches
        eng.body_generate(mfcc, label, noise)
        base = eng.launches - n0
        n1 = eng.launches
        eng.body_generate(mfcc, label, None, seeds=seeds)
        assert eng.launches - n1 == base
        n1 = eng.launches
        eng.sampler_noise(seeds, 20)
        assert eng.launches - n1 == 1
    finally:
        eng.set_pixelcnn_mode(0)


def test_errors_and_greedy(eng, ckpts):
    from talkshow_b200.engine import _ctl_struct

    aud, label = _aud(ckpts["pixel"], 2, 4, 51)
    a, lb = aud.cuda(), label.cuda()
    codes = torch.empty(2, 4, 2, dtype=torch.int64, device="cuda")
    mf = synth.synth_mfcc(2, 16, seed=5).cuda()
    poses = torch.empty(2, 16, 129, device="cuda")
    s = _lib.stream_ptr(torch.device("cuda", 0))
    sampling = _ctl_struct(0.7, 0, 1.0, 0.0, None, None)
    for ctl in (None, C.byref(sampling)):
        assert eng.L.ts_pixelcnn_sample_seeded(eng.h, _lib.ptr(a), _lib.ptr(lb), None, _lib.ptr(codes), None, 2, 4, None, 0,
                                               ctl, s) == 1
        assert eng.L.ts_body_sample_seeded(eng.h, _lib.ptr(mf), _lib.ptr(lb), None, None, _lib.ptr(poses), 2, 16, ctl, s) == 1
    sd = _seeds(2, 1).cuda()
    assert eng.L.ts_sampler_noise(eng.h, _lib.ptr(sd), None, 2, 4, 0, s) == 1
    assert eng.L.ts_sampler_noise(eng.h, _lib.ptr(sd), _lib.ptr(torch.empty(8, 2, 2048, device="cuda")), 2, 4, -1, s) == 1
    # greedy decoding runs without seeds and equals the greedy explicit call
    greedy = _ctl_struct(0.0, 0, 1.0, 0.0, None, None)
    assert eng.L.ts_pixelcnn_sample_seeded(eng.h, _lib.ptr(a), _lib.ptr(lb), None, _lib.ptr(codes), None, 2, 4, None, 0,
                                           C.byref(greedy), s) == 0
    torch.cuda.synchronize()
    assert torch.equal(codes.cpu(), eng.pixelcnn_generate(a, lb, None, temperature=0.0).cpu())
    assert eng.L.ts_body_sample_seeded(eng.h, _lib.ptr(mf), _lib.ptr(lb), None, None, _lib.ptr(poses), 2, 16,
                                       C.byref(greedy), s) == 0
    torch.cuda.synchronize()
    assert torch.equal(poses, eng.body_generate(mf, lb, None, temperature=0.0)[1])
    # the Python layer
    nz = eng.sampler_noise(sd, 4)
    for kw in [dict(seeds=sd, noise=nz), dict(seeds=None, noise=None), dict(seeds=sd.to(torch.int32), noise=None),
               dict(seeds=sd[:1], noise=None), dict(seeds=[1, 2, 3], noise=None), dict(seeds=[1.5, 2], noise=None)]:
        n = kw.pop("noise")
        with pytest.raises(ValueError):
            eng.pixelcnn_generate(a, lb, n, **kw)
        with pytest.raises(ValueError):
            eng.body_generate(mf, lb, n, **kw)
    for bad in (sd.reshape(2, 1), torch.tensor([1.0]), 5):
        with pytest.raises(ValueError):
            eng.sampler_noise(bad, 4)
    with pytest.raises(ValueError):
        eng.sampler_noise(sd, 0)


def _wrapper(e):
    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Model.vq_path = ""
    return TrainWrapper(types.SimpleNamespace(gpu=0, infer=True), cfg, engine=e)


def test_wrapper_generate_and_continuity(eng, monkeypatch):
    from talkshow_b200.engine import clip_seeds
    from talkshow_b200.nets import smplx_body_pixel as bp

    g = _wrapper(eng)
    B, M = 3, 64
    mfcc = synth.synth_mfcc(B, M, seed=81).cuda()
    label = torch.tensor([0, 1, 2])
    out = g.generate(mfcc, label, clip_seeds=77)
    _, ref = eng.body_generate(mfcc, label.cuda(), None, seeds=clip_seeds(77, B))
    assert torch.equal(out, ref) and torch.equal(g.last_codes, eng.body_generate(mfcc, label.cuda(), None, seeds=clip_seeds(77, B))[0])
    out2 = g.generate(mfcc, label, clip_seeds=[77, 78, 79], temperature=0.9, top_p=0.8, keep_logp=True)
    _, ref2, lp, kp = eng.body_generate(mfcc, label.cuda(), None, seeds=clip_seeds(77, B), temperature=0.9, top_p=0.8,
                                        want_logp=True, want_kept=True)
    assert torch.equal(out2, ref2) and torch.equal(g.last_logp, lp) and torch.equal(g.last_kept, kp)
    # continuity: a 2 s prefix, then the rest conditioned on it, both chunks seeded with the same per-clip seeds
    f0 = synth.synth_mfcc(1, 60, seed=82)[0].t().numpy()
    f1 = synth.synth_mfcc(1, 100, seed=83)[0].t().numpy()
    monkeypatch.setattr(bp, "get_mfcc_sepa", lambda *a, **k: (np.concatenate((f0, f1), 0), f0.shape[0]))
    pred = g.infer_on_audio("unused.wav", id=torch.tensor([1]), B=2, continuity=True, clip_seeds=5)
    seeds = clip_seeds(5, 2).cuda()
    lb = torch.tensor([1, 1]).cuda()
    feat = torch.from_numpy(np.concatenate((f0, f1), 0))[None].repeat(2, 1, 1)
    a0 = eng.audio_encode(feat[:, :60].transpose(1, 2).contiguous())
    a1 = eng.audio_encode(feat[:, 60:].transpose(1, 2).contiguous())
    T0, T1 = a0.shape[2], a1.shape[2]
    lat0 = torch.empty(2, T0, 2, dtype=torch.int64, device="cuda")
    lat1 = torch.empty(2, T1, 2, dtype=torch.int64, device="cuda")
    s = _lib.stream_ptr(torch.device("cuda", 0))
    assert eng.L.ts_pixelcnn_sample_seeded(eng.h, _lib.ptr(a0), _lib.ptr(lb), _lib.ptr(seeds), _lib.ptr(lat0), None, 2, T0,
                                           None, 0, None, s) == 0
    a01 = torch.cat([a0, a1], 2).contiguous()
    assert eng.L.ts_pixelcnn_sample_seeded(eng.h, _lib.ptr(a01), _lib.ptr(lb), _lib.ptr(seeds), _lib.ptr(lat1), None, 2, T1,
                                           _lib.ptr(lat0), T0, None, s) == 0
    torch.cuda.synchronize()
    assert torch.equal(g.last_codes, torch.cat([lat0, lat1], 1))
    assert pred.shape == (2, 4 * (T0 + T1), 129)
    with pytest.raises(ValueError):
        g.generate(mfcc, label, clip_seeds=1, noise_fn=lambda T, B_: None)


def test_wholebody_and_sharded(ckpts):
    from talkshow_b200.engine import Engine, clip_seeds
    from talkshow_b200.pipeline import WholeBody, shard_range

    wb = WholeBody(Engine(0))
    wb.load(ckpts["pixel"], ckpts["vq"], ckpts["face"])
    B, M = 5, 64
    mfcc = synth.synth_mfcc(B, M, seed=91).cuda()
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(92)).cuda()
    label = torch.tensor([0, 1, 2, 3, 0]).cuda()
    frame = wave.shape[1] * 30 // 16000
    try:
        outs = []
        for ob in (0, 64):                                     # sequential and overlapped paths
            wb.overlap_batch = ob
            outs.append(wb.generate(mfcc, wave, label, clip_seeds=2024))
            _, body = wb.e.body_generate(mfcc, label, None, seeds=clip_seeds(2024, B))
            face = wb.e.face_forward(wave, torch.zeros(B, 4, device="cuda"), frame)
            assert torch.equal(outs[-1], wb.e.assemble_pose(face, body)), ob
        assert torch.equal(outs[0], outs[1])
        wb.overlap_batch = 0
        one = outs[0]
        for world in (1, 2, 3):
            parts = []
            for r in range(world):
                p = wb.generate_sharded(mfcc, wave, label, r, world, gather=False, clip_seeds=2024)
                lo, hi = shard_range(B, r, world)
                assert torch.equal(p, one[lo:hi]), (world, r)              # each shard is the rows of the single call
                parts.append(p)
            assert torch.equal(torch.cat(parts), one), world
    finally:
        torch.cuda.synchronize()
        wb.close()
        wb.e.close()
