"""GPU (-m gpu): anchored sampling of the body prior (ts_pixelcnn_sample_anchored, ts_body_sample_anchored) on every sampler
executor of test_gpu_seeded.CONFIGS and on the 6-D prior, with explicit noise and with seeds.

The rule is pinned by invariants that hold bit for bit: anchors that pin nothing give the existing call; pinning draws to
the codes they draw anyway changes nothing (log p included: a pinned draw's log p is the tail of a sampled one); a pinned
prefix is the pre_latents call.  The oracle check is that of test_gpu_seeded: the oracle's draw on teacher-forced logits of
the engine's own codes, with every pinned draw replaced by its anchor (tests/oracle_anchored.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import talkshow_oracle as O
from conftest import GOLDEN, ROOT
from talkshow_b200 import _lib, synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_anchored as OA  # noqa: E402
import oracle_sampling as OSM  # noqa: E402
import oracle_seeded as OS  # noqa: E402
from test_gpu_seeded import CONFIGS, SETTINGS, _aud, _engine, _seeds, _wrapper, config, eng, six  # noqa: E402,F401

pytestmark = pytest.mark.gpu
SOURCES = ("noise", "seeds")


def _run(e, aud, label, s, src, seeds, noise, anchors=None, want_logits=False, **kw):
    """[codes, logp, kept, logits] of one call (None where the call has none); s None: the default draw"""
    greedy = s is not None and s["temperature"] == 0
    n = None if greedy or src != "noise" else noise
    sd = None if greedy or src != "seeds" else seeds
    if anchors is not None:
        kw["anchors"] = anchors
    if s is None:
        out = e.pixelcnn_generate(aud, label, n, seeds=sd, want_logits=want_logits, **kw)
        out = list(out) if want_logits else [out]
        return [out[0].cpu(), None, None, out[1].cpu() if want_logits else None]
    want_kept = "top_p" in s
    out = [x.cpu() for x in e.pixelcnn_generate(aud, label, n, seeds=sd, want_logp=True, want_kept=want_kept,
                                                  want_logits=want_logits, **s, **kw)]
    logits = out.pop(1) if want_logits else None
    return [out[0], out[1], out[2] if want_kept else None, logits]


def _equal(a, b, what):
    for x, y, n in zip(a, b, ("codes", "logp", "kept", "logits")):
        if x is not None or y is not None:
            assert x is not None and y is not None and x.shape == y.shape, (what, n)
            bad = x != y
            assert not bad.any(), (what, n, int(bad.sum()), bad.nonzero()[:4].tolist(), x[bad][:4].tolist(), y[bad][:4].tolist())


def _skip_tile(config, B):
    if B > 16 and config.startswith("m0-t16") or B > 32 and config.startswith("m0-t32"):
        pytest.skip("tile smaller than the batch")


def _masks(B, T, seed):
    """pin patterns [B,T,2] bool: a random half, a window, column 1 only, everything"""
    g = torch.Generator().manual_seed(seed)
    half = torch.rand(B, T, 2, generator=g) < 0.5
    win = torch.zeros(B, T, 2, dtype=torch.bool)
    win[:, T // 4: T // 4 + max(1, T // 3)] = True
    col = torch.zeros(B, T, 2, dtype=torch.bool)
    col[..., 1] = True
    return {"half": half, "window": win, "column": col, "all": torch.ones(B, T, 2, dtype=torch.bool)}


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
@pytest.mark.parametrize("B,T", [(64, 75), (12, 75), (1, 30), (100, 12)])
def test_unpinned_equals_existing(eng, ckpts, config, B, T):
    _skip_tile(config, B)
    aud, label = _aud(ckpts["pixel"], B, T, 100 + B)
    seeds = _seeds(B, B + T)
    noise = eng.sampler_noise(seeds, T)
    free = torch.full((B, T, 2), -1, dtype=torch.int64)
    for src in SOURCES:
        for s in SETTINGS:
            n0 = eng.launches
            ref = _run(eng, aud, label, s, src, seeds, noise, want_logits=True)
            n1 = eng.launches
            got = _run(eng, aud, label, s, src, seeds, noise, anchors=free, want_logits=True)
            assert eng.launches - n1 == n1 - n0, (config, s, src)
            _equal(got, ref, (config, B, T, s, src))


def test_unpinned_equals_existing_6d(six, monkeypatch):
    e, ck, _ = six
    for mb in ("4", "8"):
        monkeypatch.setenv("TS_PIX3_MB", mb)
        for B, T in [(64, 10), (12, 10), (1, 10)]:
            aud, label = _aud(ck, B, T, 300 + B)
            seeds = _seeds(B, B)
            noise = e.sampler_noise(seeds, T)
            free = torch.full((B, T, 2), -1, dtype=torch.int64)
            for src in SOURCES:
                for s in SETTINGS:
                    got, ref = _run(e, aud, label, s, src, seeds, noise, anchors=free), _run(e, aud, label, s, src, seeds, noise)
                    # codes and keep sets bit for bit; log p to 1e-5: two identical calls of the 6-D cluster kernel at 4
                    # samples per cluster have been seen to differ in the last bits of log p with every code equal
                    # (DESIGN §3d), so a bitwise log p check here would test that, not the anchors
                    _equal([got[0], None, got[2]], [ref[0], None, ref[2]], (mb, B, T, s, src))
                    if ref[1] is not None:
                        assert (got[1] - ref[1]).abs().max() <= 1e-5, (mb, B, T, s, src)


def _pin_own(e, aud, label, settings, seeds, noise, seed):
    B, T = aud.shape[0], aud.shape[2]
    for src in SOURCES:
        for s in settings:
            ref = _run(e, aud, label, s, src, seeds, noise)
            for name, m in _masks(B, T, seed).items():
                got = _run(e, aud, label, s, src, seeds, noise, anchors=torch.where(m, ref[0], -1))
                what = (s, src, name)
                assert torch.equal(got[0], ref[0]), what
                if ref[1] is not None:
                    assert torch.equal(got[1], ref[1]), what
                if ref[2] is not None:
                    assert torch.equal(got[2][~m], ref[2][~m]) and (got[2][m] == 0).all(), what


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_pin_own_codes(eng, ckpts, config):
    aud, label = _aud(ckpts["pixel"], 12, 40, 61)
    seeds = _seeds(12, 6)
    noise = eng.sampler_noise(seeds, 40)
    settings = [dict(temperature=1.0, top_k=0)] + SETTINGS[1:]
    _pin_own(eng, aud, label, settings, seeds, noise, 62)


def test_pin_own_codes_6d(six, monkeypatch):
    e, ck, _ = six
    for mb in ("4", "8"):
        monkeypatch.setenv("TS_PIX3_MB", mb)
        aud, label = _aud(ck, 12, 10, 63)
        seeds = _seeds(12, 7)
        _pin_own(e, aud, label, [dict(temperature=1.0, top_k=0)] + SETTINGS[1:], seeds, e.sampler_noise(seeds, 10), 64)


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_pin_own_codes_body_generate(eng, six, geo):
    e = eng if geo == "3d" else six[0]
    B, M = 12, 64
    mfcc = synth.synth_mfcc(B, M, seed=65).cuda()
    label = (torch.arange(B) % 4).cuda()
    seeds = _seeds(B, 8)
    noise = e.sampler_noise(seeds, M // 4)
    for kw in (dict(noise=noise), dict(noise=None, seeds=seeds), dict(noise=noise, temperature=0.8, top_k=64, want_logp=True)):
        kw = dict(kw)
        n = kw.pop("noise")
        ref = e.body_generate(mfcc, label, n, **kw)
        for name, m in _masks(B, M // 4, 66).items():
            got = e.body_generate(mfcc, label, n, anchors=torch.where(m.cuda(), ref[0], -1), **kw)
            for x, y in zip(got, ref):
                assert torch.equal(x, y), (geo, name, kw.keys())


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_pinned_prefix_equals_pre_latents(eng, ckpts, config):
    B, T0, T = 5, 6, 10
    aud, label = _aud(ckpts["pixel"], B, T0 + T, 41)
    pre = torch.randint(0, 2048, (B, T0, 2), generator=torch.Generator().manual_seed(42))
    seeds = _seeds(B, 4)
    anchors = torch.cat([pre, torch.full((B, T, 2), -1, dtype=torch.int64)], 1)
    for s in (None, SETTINGS[1], SETTINGS[4], SETTINGS[-2]):
        ref = _run(eng, aud, label, s, "seeds", seeds, None, T=T, pre_latents=pre)
        got = _run(eng, aud, label, s, "seeds", seeds, None, anchors=anchors)
        assert torch.equal(got[0][:, :T0], pre), (config, s)
        for x, y, n in zip(got[:3], ref[:3], ("codes", "logp", "kept")):
            if y is not None:
                assert torch.equal(x[:, T0:], y), (config, s, n)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_everything_pinned(eng, ckpts, config):
    B, T = 12, 30
    aud, label = _aud(ckpts["pixel"], B, T, 71)
    anchors = torch.randint(0, 2048, (B, T, 2), generator=torch.Generator().manual_seed(72))
    seeds = _seeds(B, 9)
    noise = eng.sampler_noise(seeds, T)
    for src in SOURCES:
        for s in (dict(temperature=1.0, top_k=0), SETTINGS[4], SETTINGS[-3]):
            codes, logp, kept, logits = _run(eng, aud, label, s, src, seeds, noise, anchors=anchors, want_logits=True)
            assert torch.equal(codes, anchors), (config, s, src)
            ref = torch.log_softmax(logits.double(), -1).reshape(T, 2, B, 2048).permute(2, 0, 1, 3)
            ref = ref.gather(-1, anchors.unsqueeze(-1)).squeeze(-1)
            assert (logp.double() - ref).abs().max() <= 1e-5, (config, s, src)
            if kept is not None:
                assert (kept == 0).all()
    nll = eng.pixelcnn_score(aud, label, anchors).cpu()
    assert (logp + nll).abs().mean() <= 2.5e-5
    eng.set_tensor_cores(0)
    try:
        assert (logp + eng.pixelcnn_score(aud, label, anchors).cpu()).abs().max() <= 1e-4
    finally:
        eng.set_tensor_cores(6)


def _random_anchors(B, T, seed, frac=0.3):
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, 2048, (B, T, 2), generator=g)
    return torch.where(torch.rand(B, T, 2, generator=g) < frac, codes, -1)


@pytest.mark.parametrize("B,T", [(64, 75), (12, 75), (1, 30), (100, 12)])
def test_codes_equal_oracle(eng, ckpts, monkeypatch, B, T):
    aud, label = _aud(ckpts["pixel"], B, T, 500 + B)
    seeds = _seeds(B, 5)
    anchors = _random_anchors(B, T, B + T)
    codes = eng.pixelcnn_generate(aud, label, None, seeds=seeds, anchors=anchors).cpu()
    noise = torch.from_numpy(OS.noise(seeds.tolist(), T))
    assert torch.equal(OA.teacher_forced_draw(ckpts["pixel"]["generator"], codes, label, aud, noise, anchors), codes)
    # every executor gives those codes
    for name, mode, env in CONFIGS:
        if B > 16 and name == "m0-t16" or B > 32 and name == "m0-t32" or mode == 1 and B * T > 1000:
            continue
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng.set_pixelcnn_mode(mode)
        try:
            assert torch.equal(eng.pixelcnn_generate(aud, label, None, seeds=seeds, anchors=anchors).cpu(), codes), name
        finally:
            eng.set_pixelcnn_mode(0)


def test_codes_equal_oracle_6d(six):
    e, ck, _ = six
    B, T = 12, 10
    aud, label = _aud(ck, B, T, 501)
    seeds = _seeds(B, 5)
    anchors = _random_anchors(B, T, 77)
    codes = e.pixelcnn_generate(aud, label, None, seeds=seeds, anchors=anchors).cpu()
    noise = torch.from_numpy(OS.noise(seeds.tolist(), T))
    assert torch.equal(OA.teacher_forced_draw(ck["generator"], codes, label, aud, noise, anchors), codes)


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_reference_fixture(eng, six, geo):
    path = os.path.join(GOLDEN, "anchored.npz")
    z = np.load(path)
    e = eng if geo == "3d" else six[0]
    pre = geo + "_"
    mfcc = torch.from_numpy(z[pre + "mfcc"])
    label = torch.from_numpy(z[pre + "label"])
    stride = int(z[pre + "pose_stride"])
    B, T = z[pre + "codes"].shape[1:3]
    for i, name in enumerate(str(n) for n in z[pre + "cases"]):
        t, k, p = (float(v) for v in z[pre + "setting"][i])
        anchors = torch.from_numpy(z[pre + "anchors"][i])
        noise = OSM.reference_noise(int(z[pre + "seed"][i]), 2 * T, B)
        kw = dict(temperature=t, top_k=int(k), top_p=p, want_logp=True)
        codes, poses, logp = e.body_generate(mfcc, label, noise, anchors=anchors, **kw)[:3]
        assert torch.equal(codes.cpu(), torch.from_numpy(z[pre + "codes"][i])), (geo, name)
        # the oracle's (and the engine's) logits agree with the reference's to ~1e-5: log p is compared at that level
        assert (logp.cpu() - torch.from_numpy(z[pre + "logp"][i])).abs().max() <= 5e-5, (geo, name)
        err = (poses.cpu()[:, ::stride] - torch.from_numpy(z[pre + "poses"][i])).abs().max().item()
        assert err <= 1e-4, (geo, name, err)


def _batch_position(e, aud, label, M_mfcc=None):
    B, T = aud.shape[0], aud.shape[2]
    seeds = _seeds(B, 9)
    anchors = _random_anchors(B, T, 91, 0.5)
    for b in (0, 7, 11):
        seeds[b] = 424242
        anchors[b] = anchors[0]
    for s in (dict(temperature=1.0, top_k=0), SETTINGS[4], SETTINGS[-3]):
        full = _run(e, aud, label, s, "seeds", seeds, None, anchors=anchors)
        for b in (0, 7, 11):
            one = _run(e, aud[b:b + 1], label[b:b + 1], s, "seeds", seeds[b:b + 1], None, anchors=anchors[b:b + 1])
            assert torch.equal(one[0][0], full[0][b]) and torch.equal(one[1][0], full[1][b]), (s, b)


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_batch_position(eng, ckpts, config):
    aud, label = _aud(ckpts["pixel"], 12, 16, 31)
    _batch_position(eng, aud, label)


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_batch_position_body(eng, six, geo):
    e = eng if geo == "3d" else six[0]
    if geo == "6d":
        aud, label = _aud(six[1], 12, 10, 33)
        _batch_position(e, aud, label)
    B, M = 12, 64
    mfcc = synth.synth_mfcc(B, M, seed=71).cuda()
    label = (torch.arange(B) % 4).cuda()
    seeds = _seeds(B, 3)
    anchors = _random_anchors(B, M // 4, 92, 0.5)
    codes, poses = e.body_generate(mfcc, label, None, seeds=seeds, anchors=anchors)
    for b in (0, 7, 11):
        c1, p1 = e.body_generate(mfcc[b:b + 1], label[b:b + 1], None, seeds=seeds[b:b + 1], anchors=anchors[b:b + 1])
        assert torch.equal(c1[0], codes[b]) and torch.equal(p1[0], poses[b]), b


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_pose_recipe(eng, six, geo):
    """pin every draw to the codes of known poses: the result is the VQ decoding of those codes"""
    e = eng if geo == "3d" else six[0]
    B, M = 4, 64
    mfcc = synth.synth_mfcc(B, M, seed=95).cuda()
    label = (torch.arange(B) % 4).cuda()
    _, known = e.body_generate(mfcc, label, None, seeds=_seeds(B, 11))
    known = known + 0.01 * torch.randn(known.shape, generator=torch.Generator().manual_seed(96)).cuda()
    nb = e.vq_dim(0)
    codes = torch.stack([e.vq_encode(0, known[..., :nb].contiguous()), e.vq_encode(1, known[..., nb:].contiguous())], -1)
    got_codes, poses = e.body_generate(mfcc, label, None, seeds=_seeds(B, 12), anchors=codes)
    assert torch.equal(got_codes, codes)
    ref = torch.cat([e.vq_decode(0, codes[..., 0].contiguous()), e.vq_decode(1, codes[..., 1].contiguous())], 1).transpose(1, 2)
    assert torch.equal(poses, ref)


def test_wrappers(eng, monkeypatch):
    from talkshow_b200.engine import clip_seeds
    from talkshow_b200.nets import smplx_body_pixel as bp

    g = _wrapper(eng)
    B, M = 3, 64
    T = M // 4
    mfcc = synth.synth_mfcc(B, M, seed=81).cuda()
    label = torch.tensor([0, 1, 2])
    anchors = _random_anchors(B, T, 82, 0.5)
    out = g.generate(mfcc, label, clip_seeds=77, anchors=anchors.numpy())
    c, ref = eng.body_generate(mfcc, label.cuda(), None, seeds=clip_seeds(77, B), anchors=anchors)
    assert torch.equal(out, ref) and torch.equal(g.last_codes, c)
    # keep the hands of that clip, resample the body
    keep_hands = torch.where(torch.arange(2) == 1, g.last_codes.cpu(), -1)
    g.generate(mfcc, label, clip_seeds=78, anchors=keep_hands)
    assert torch.equal(g.last_codes[..., 1], c[..., 1])
    # infer: anchors over the chunk's rows, composed with pre_latents
    feat = synth.synth_mfcc(B, M, seed=83).transpose(1, 2).contiguous()
    lat0, a0, _, _ = g.infer(feat, 0, label, B, clip_seeds=5)
    lat1, _, body, hand = g.infer(feat, 0, label, B, lat0, a0, None, clip_seeds=5, anchors=anchors)
    a1 = eng.audio_encode(feat.transpose(1, 2).contiguous())
    ref1 = eng.pixelcnn_generate(torch.cat([a0[..., 0], a1], 2), label.cuda(), None, T=T, pre_latents=lat0,
                                 seeds=clip_seeds(5, B), anchors=anchors)
    assert torch.equal(lat1, ref1)
    assert torch.equal(body, eng.vq_decode(0, lat1[..., 0].contiguous()))
    monkeypatch.setattr(bp, "get_mfcc_sepa", lambda *a, **k: (np.zeros((160, 64), np.float32), 60))
    with pytest.raises(ValueError):
        g.infer_on_audio("unused.wav", B=1, continuity=True, anchors=anchors[:1])
    f = synth.synth_mfcc(1, M, seed=84)[0].t().numpy()
    pred = g.infer_on_audio(f, B=1, clip_seeds=3, anchors=anchors[:1])
    assert torch.equal(g.last_codes.cpu()[anchors[:1] >= 0], anchors[:1][anchors[:1] >= 0])
    assert pred.shape == (1, M, 129)


def test_wholebody_and_sharded(ckpts):
    from talkshow_b200.engine import Engine, clip_seeds
    from talkshow_b200.pipeline import WholeBody, shard_range

    wbs = [WholeBody(Engine(0)), WholeBody(Engine(0))]
    for wb in wbs:
        wb.load(ckpts["pixel"], ckpts["vq"], ckpts["face"])
    wb = wbs[0]
    B, M = 5, 64
    mfcc = synth.synth_mfcc(B, M, seed=91).cuda()
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(92)).cuda()
    label = torch.tensor([0, 1, 2, 3, 0]).cuda()
    frame = wave.shape[1] * 30 // 16000
    anchors = _random_anchors(B, M // 4, 93, 0.4)
    try:
        outs = []
        for ob in (0, 64):                                     # sequential and overlapped paths
            wb.overlap_batch = ob
            outs.append(wb.generate(mfcc, wave, label, clip_seeds=2024, anchors=anchors, keep_codes=True))
            codes, body = wb.e.body_generate(mfcc, label, None, seeds=clip_seeds(2024, B), anchors=anchors)
            assert torch.equal(wb.last_codes, codes), ob
            face = wb.e.face_forward(wave, torch.zeros(B, 4, device="cuda"), frame)
            assert torch.equal(outs[-1], wb.e.assemble_pose(face, body)), ob
            # anchored noise-driven call, and the default call keeps no codes
            n = wb.e.sampler_noise(clip_seeds(7, B), M // 4)
            wb.generate(mfcc, wave, label, noise=n, anchors=anchors.cuda(), keep_codes=True)
            assert torch.equal(wb.last_codes, wb.e.body_generate(mfcc, label, n, anchors=anchors)[0]), ob
            wb.generate(mfcc, wave, label, noise=n)
            assert wb.last_codes is None
        assert torch.equal(outs[0], outs[1])
        for w in wbs:
            w.overlap_batch = 0
        parts = []
        for r in range(2):                                     # world 2 on two engines
            p = wbs[r].generate_sharded(mfcc, wave, label, r, 2, gather=False, clip_seeds=2024, anchors=anchors)
            lo, hi = shard_range(B, r, 2)
            assert torch.equal(p, outs[0][lo:hi]), r
            parts.append(p)
        assert torch.equal(torch.cat(parts), outs[0])
    finally:
        torch.cuda.synchronize()
        for w in wbs:
            w.close()
            w.e.close()


def test_errors(eng, ckpts):
    from talkshow_b200.engine import _ctl_struct

    aud, label = _aud(ckpts["pixel"], 2, 4, 51)
    a, lb = aud.cuda(), label.cuda()
    codes = torch.empty(2, 4, 2, dtype=torch.int64, device="cuda")
    mf = synth.synth_mfcc(2, 16, seed=5).cuda()
    poses = torch.empty(2, 16, 129, device="cuda")
    s = _lib.stream_ptr(torch.device("cuda", 0))
    sd = _seeds(2, 1).cuda()
    nz = eng.sampler_noise(sd, 4)
    anc = torch.full((2, 4, 2), 5, dtype=torch.int64, device="cuda")      # every draw pinned: still one noise source
    sampling = _ctl_struct(0.7, 0, 1.0, 0.0, None, None)
    greedy = _ctl_struct(0.0, 0, 1.0, 0.0, None, None)
    bad_ctl = _ctl_struct(-1.0, 0, 1.0, 0.0, None, None)
    P = lambda n, sd_, ctl, anchors=anc: eng.L.ts_pixelcnn_sample_anchored(  # noqa: E731
        eng.h, _lib.ptr(a), _lib.ptr(lb), _lib.ptr(n), _lib.ptr(sd_), _lib.ptr(anchors), _lib.ptr(codes), None, 2, 4, None, 0,
        ctl, s)
    Bd = lambda n, sd_, ctl, anchors=anc: eng.L.ts_body_sample_anchored(  # noqa: E731
        eng.h, _lib.ptr(mf), _lib.ptr(lb), _lib.ptr(n), _lib.ptr(sd_), _lib.ptr(anchors), None, _lib.ptr(poses), 2, 16, ctl, s)
    for fn in (P, Bd):
        for ctl in (None, C.byref(sampling)):
            assert fn(None, None, ctl) == 1
            assert fn(nz, sd, ctl) == 1
        assert fn(nz, None, C.byref(bad_ctl)) == 1
        assert fn(None, None, C.byref(greedy)) == 0
        assert fn(nz, None, None) == 0 and fn(None, sd, C.byref(sampling)) == 0
    assert eng.L.ts_pixelcnn_sample_anchored(eng.h, _lib.ptr(a), _lib.ptr(lb), _lib.ptr(nz), None, _lib.ptr(anc),
                                             _lib.ptr(codes), None, 0, 4, None, 0, None, s) == 1
    torch.cuda.synchronize()
    assert (codes == 5).all()
    # out-of-range device values sample (the kernel never gathers outside the table): equal to -1
    junk = torch.tensor([-7, 2048, 1 << 40, -1], dtype=torch.int64).repeat(4).reshape(2, 4, 2).cuda()
    assert P(nz, None, None, junk) == 0
    torch.cuda.synchronize()
    assert torch.equal(codes, eng.pixelcnn_generate(a, lb, nz))
    # the Python layer
    for bad in (torch.zeros(2, 4, 2, dtype=torch.int32), torch.zeros(2, 4, dtype=torch.int64), torch.zeros(2, 5, 2, dtype=torch.int64),
                torch.full((2, 4, 2), 2048, dtype=torch.int64), torch.full((2, 4, 2), -2, dtype=torch.int64).cuda(),
                np.zeros((2, 4, 2), np.float32), [[[0, 0]] * 4] * 2):
        with pytest.raises(ValueError):
            eng.pixelcnn_generate(a, lb, nz, anchors=bad)
        with pytest.raises(ValueError):
            eng.body_generate(mf, lb, nz, anchors=bad)
