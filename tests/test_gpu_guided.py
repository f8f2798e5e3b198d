"""GPU (-m gpu): guided sampling of the body prior (ts_pixelcnn_sample_guided, ts_body_sample_guided) on every sampler
executor of test_gpu_seeded.CONFIGS and on the 6-D prior, with explicit noise and with seeds.

Pinned bit for bit: the reference fixture (tests/golden/guided.npz, tests/golden/make_golden_guided.py); at w = 1 a pair draws the codes, conditional log p and keep sizes of the shaped call on its clip alone
(per-clip controls, penalties and a ban list included); both branches of a pair write the same codes and keep sizes; the
oracle's guided draw (tests/oracle_guided.py) on the engine's own raw logits of both branches gives the engine's code; a
pair alone equals the same pair in a mixed batch.  Each branch's log p equals -nll of the teacher-forced scorer under that
branch's conditioning within the bars of the shaped tests.  Cluster-executor log p of separate calls is compared at 1e-5
(the open issue of DESIGN §3d)."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from talkshow_b200 import _lib, synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_guided as OG  # noqa: E402
import oracle_nucleus as ON  # noqa: E402
import oracle_shaped as OSH  # noqa: E402
from test_gpu_clip_ctl import GROUPS, SHAPES, SOURCES, _equal, _gen, _per_clip, _tol  # noqa: E402
from test_gpu_seeded import CONFIGS, _aud, _engine, _seeds, config, eng, six  # noqa: E402,F401
from test_gpu_shaped import SHAPING, _ban, _shaping  # noqa: E402
from test_guided_cpu import fixture_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
SCALES = [1.0, 2.0, 0.5, 3.0, 1.5]


def _skip_tile(config, B):
    nb = 2 * min(B, 32)   # branches per launch
    if nb > 16 and config.startswith("m0-t16") or nb > 32 and config.startswith("m0-t32"):
        pytest.skip("tile smaller than the launch")


def _guided(e, aud, label, gaud, src, noise, seeds, sampled=True, **kw):
    """codes, logp, kept, negative log p of one guided call"""
    s = dict(noise=None, seeds=None) if not sampled else (dict(noise=noise, seeds=None) if src == "noise"
                                                          else dict(noise=None, seeds=seeds))
    out = e.pixelcnn_generate(aud, label, s["noise"], seeds=s["seeds"], want_logp=True, want_kept=True,
                              want_guide_logp=True, guide_aud=gaud, **kw)
    return [x.cpu() for x in out]


def _check_identity(e, ck, B, T, src, tol, what, seed):
    aud, label = _aud(ck, B, T, seed)
    gaud = _aud(ck, B, T, seed + 1)[0]
    seeds = _seeds(B, seed)
    noise = e.sampler_noise(seeds, T).cpu()
    pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, seed)
    # unshaped: the per-clip call's log p may take draw_controlled's sum_raw shortcut, the guided one never does
    _equal(_guided(e, aud, label, gaud, src, noise, seeds, guidance=1.0, **pc)[:3], _gen(e, aud, label, src, noise, seeds, **pc),
           (what, "w = 1, unshaped"), tol)
    ref = _gen(e, aud, label, src, noise, seeds, code_bias=bias, **pc, **sh)
    got = _guided(e, aud, label, gaud, src, noise, seeds, guidance=1.0, code_bias=bias, **pc, **sh)
    _equal(got[:3], ref, (what, "w = 1"), tol)
    # the negative audio does not matter at w = 1, and does at w != 1
    other = _guided(e, aud, label, aud.flip(-1).contiguous(), src, noise, seeds, guidance=1.0, code_bias=bias, **pc, **sh)
    _equal(other[:3], ref, (what, "w = 1, other negative"), tol)
    w2 = _guided(e, aud, label, gaud, src, noise, seeds, guidance=3.0, code_bias=bias, **pc, **sh)[0]
    w2b = _guided(e, aud, label, aud.flip(-1).contiguous(), src, noise, seeds, guidance=3.0, code_bias=bias, **pc, **sh)[0]
    assert not torch.equal(w2, w2b) and not torch.equal(w2, ref[0]), what
    assert not (bias.gather(-1, w2.transpose(1, 2)) == float("-inf")).any(), (what, "banned code drawn")


@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_identity_at_w1(eng, ckpts, config, B, T, src):
    _skip_tile(config, B)
    _check_identity(eng, ckpts["pixel"], B, T, src, _tol(config), (config, B, T, src), 1700 + B)


@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("mb", ["4", "8"])
def test_identity_at_w1_6d(six, monkeypatch, mb, B, T, src):
    e, ck, _ = six
    monkeypatch.setenv("TS_PIX3_MB", mb)
    _check_identity(e, ck, B, T, src, 1e-5, ("6d", mb, B, T, src), 1800 + B)


def _run_fixture(e, z, case):
    """the engine's codes and keep sizes on fixture case ``case`` (tests/golden/guided.npz)"""
    f = fixture_inputs(z, case)
    kw = dict(f["kw"], want_kept=True, guidance=f["guidance"], guide_label=f["glabel"], guide_style=f["gstyle"])
    if f["pre"] is not None:
        aud = torch.cat([e.audio_encode(f["mpre"]), e.audio_encode(f["mfcc"])], 2)
        gaud = torch.cat([e.audio_encode(f["gmpre"]), e.audio_encode(f["gmfcc"])], 2)
        codes, kept = e.pixelcnn_generate(aud, f["label"], f["noise"], T=f["T"], pre_latents=f["pre"], guide_aud=gaud, **kw)
    else:
        codes, _, kept = e.body_generate(f["mfcc"], f["label"], f["noise"], guide_mfcc=f["gmfcc"], **kw)
    return codes.cpu(), kept.cpu()


@pytest.mark.parametrize("case", ["3d", "style", "pre"])
@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_reference_fixture(eng, config, case):
    """the reference, run on 2P interleaved rows with both branches fed the guided code, draws the engine's codes and
    keep sizes bit for bit (every draw's nucleus and min-p margin is at least 1e-5)"""
    z = np.load(os.path.join(GOLDEN, "guided.npz"))
    _skip_tile(config, len(z["settings"]))
    codes, kept = _run_fixture(eng, z, case)
    assert torch.equal(codes, torch.from_numpy(z["codes_%s" % case])), (config, case)
    assert torch.equal(kept, torch.from_numpy(z["kept_%s" % case])), (config, case)


@pytest.mark.parametrize("mb", ["4", "8"])
def test_reference_fixture_6d(six, monkeypatch, mb):
    z = np.load(os.path.join(GOLDEN, "guided.npz"))
    monkeypatch.setenv("TS_PIX3_MB", mb)
    codes, kept = _run_fixture(six[0], z, "6d")
    assert torch.equal(codes, torch.from_numpy(z["codes_6d"])) and torch.equal(kept, torch.from_numpy(z["kept_6d"])), mb


def _oracle_on_logits(codes, kept, logits, noise, pc, sh, bias, w, what):
    """every sampled draw equals the oracle's guided draw on the engine's raw logits of both branches; draws whose nucleus
    or min-p keep set lies within 1e-5 of changing are skipped (the margin rule of the nucleus tests)"""
    B, T = codes.shape[:2]
    n = 0
    for i in range(T):
        for j in range(2):
            lg = logits[2 * i + j]
            for b in range(B):
                t, k, p, m = (pc[key][b] for key in ("temperature", "top_k", "top_p", "min_p"))
                th, win = sh["repetition_penalty"][b], sh["repetition_window"][b]
                g = OSH.shape(OG.guided_logits(lg[2 * b], lg[2 * b + 1], w[b]), codes[b, max(0, i - win):i, j], th,
                              bias[b, j])[None]
                if t > 0 and (p < 1.0 or m > 0.0):
                    _, mp, mm = ON.keep_mask(g, t, k, p, m, return_margin=True)
                    if min(float(mp[0]), float(mm[0])) < 1e-5:
                        continue
                code, kn = OSH.draw(g, None if t == 0 else noise[2 * i + j][b:b + 1], t, k, p, m)
                assert int(code[0]) == int(codes[b, i, j]) and int(kn[0]) == int(kept[b, i, j]), (what, b, i, j)
                n += 1
    assert n >= B * T


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_oracle_on_engine_logits_and_pair_alone(eng, ckpts, config):
    B, T = 8, 16
    ck = ckpts["pixel"]
    aud, label = _aud(ck, B, T, 41)
    gaud = _aud(ck, B, T, 42)[0]
    seeds = _seeds(B, 41)
    noise = eng.sampler_noise(seeds, T).cpu()
    pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, 44)
    w = [SCALES[b % len(SCALES)] for b in range(B)]
    glabel = (label + 1) % 4
    codes, logits, logp, kept, glogp = (x.cpu() for x in eng.pixelcnn_generate(
        aud, label, noise, want_logits=True, want_logp=True, want_kept=True, want_guide_logp=True, guidance=w,
        guide_aud=gaud, guide_label=glabel, code_bias=bias, **pc, **sh))
    _oracle_on_logits(codes, kept, logits, noise, pc, sh, bias, w, config)
    # each branch's log p is that of its own raw prior on the guided codes
    nll = eng.pixelcnn_score(aud, label, codes).cpu()
    gnll = eng.pixelcnn_score(gaud, glabel, codes).cpu()
    for lp, nl in ((logp, nll), (glogp, gnll)):
        assert (lp + nl).abs().mean() <= 2.5e-5 and (lp + nl).abs().max() <= 1e-4, config
    # a pair alone equals the same pair inside the mixed batch
    tol = _tol(config)
    for b in (0, 3, B - 1):
        s = GROUPS[b % len(GROUPS)]
        th, win = SHAPING[b % len(SHAPING)]
        one = eng.pixelcnn_generate(aud[b:b + 1], label[b:b + 1], noise[:, b:b + 1] if s["temperature"] > 0 else None,
                                    want_logp=True, want_kept=True, want_guide_logp=True, guidance=w[b],
                                    guide_aud=gaud[b:b + 1], guide_label=glabel[b:b + 1], code_bias=bias[b],
                                    repetition_penalty=th, repetition_window=win, **s)
        one = [x.cpu() for x in one]
        _equal([codes[b:b + 1], logp[b:b + 1], kept[b:b + 1]], one[:3], (config, "alone", b), tol)
        assert (glogp[b:b + 1] - one[3]).abs().max() <= tol, (config, "alone", b)


def test_oracle_on_engine_logits_6d(six, monkeypatch):
    e, ck, _ = six
    B, T = 8, 10
    aud, label = _aud(ck, B, T, 45)
    seeds = _seeds(B, 45)
    noise = e.sampler_noise(seeds, T).cpu()
    pc, sh, bias = _per_clip(B), _shaping(B), _ban(B, 46)
    w = [SCALES[b % len(SCALES)] for b in range(B)]
    for mb in ("4", "8"):
        monkeypatch.setenv("TS_PIX3_MB", mb)
        codes, logits, kept = (x.cpu() for x in e.pixelcnn_generate(
            aud, label, noise, want_logits=True, want_kept=True, guidance=w, guide_label=(label + 2) % 4, code_bias=bias,
            **pc, **sh))
        _oracle_on_logits(codes, kept, logits, noise, pc, sh, bias, w, ("6d", mb))


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=[c[0] for c in CONFIGS])
def test_c_abi_pairs(eng, ckpts, config):
    """the raw entry point: both branches of a pair write the same codes and keep sizes, each branch's log p is its own;
    pre_latents and anchors are per pair; bad scales are refused naming the pair"""
    P, T0, T = 4, 3, 8
    aud, label = _aud(ckpts["pixel"], 2 * P, T0 + T, 91)
    aud, label = aud.cuda(), label.cuda()
    seeds = _seeds(P, 91).cuda()
    pre = torch.randint(0, 2048, (P, T0, 2), generator=torch.Generator().manual_seed(92)).cuda()
    anchors = torch.full((P, T, 2), -1, dtype=torch.int64)
    anchors[:, 2, 1] = torch.arange(P) * 5
    anchors = anchors.cuda()
    L, h, p = eng.L, eng.h, _lib.ptr
    s = _lib.stream_ptr(eng.device)
    idx = torch.empty(2 * P, T, 2, dtype=torch.int64, device=eng.device)
    logp = torch.empty(2 * P, T, 2, device=eng.device)
    kept = torch.empty(2 * P, T, 2, dtype=torch.int32, device=eng.device)
    ctl = _lib.ts_sample_ctl(0.9, 0, 1.0, 0.0, logp.data_ptr(), kept.data_ptr())

    def sample(w):
        wa = np.asarray(w, np.float32)
        rc = L.ts_pixelcnn_sample_guided(h, p(aud), p(label), None, 4, None, p(seeds), p(anchors), p(idx), None, P, T, p(pre),
                                         T0, ctl, None, None, None, wa.ctypes.data, s)
        torch.cuda.synchronize()
        return rc

    assert sample([1.0, 2.0, 0.0, 100.0]) == 0
    c, lp, k = idx.cpu(), logp.cpu(), kept.cpu()
    assert torch.equal(c[0::2], c[1::2]) and torch.equal(k[0::2], k[1::2])
    assert torch.equal(c[0::2, 2, 1], torch.arange(P) * 5) and (k[:, 2, 1] == 0).all()
    pre2 = pre.cpu().repeat_interleave(2, 0)
    nll = eng.pixelcnn_score(aud, label, torch.cat([pre2, c], 1)).cpu()[:, T0:]
    assert (lp + nll).abs().mean() <= 2.5e-5 and (lp + nll).abs().max() <= 1e-4, config
    for bad in ([1.0, -0.1, 1.0, 1.0], [1.0, 1.0, float("nan"), 1.0], [1.0, 1.0, 1.0, 100.5], [float("inf")] * 4):
        assert sample(bad) == 1
        pair = [i for i, v in enumerate(bad) if not (np.isfinite(v) and 0 <= v <= 100)][0]
        assert b"pair %d" % pair in L.ts_last_error(h)
    assert L.ts_pixelcnn_sample_guided(h, p(aud), p(label), None, 4, None, p(seeds), None, p(idx), None, 0, T, None, 0, ctl,
                                       None, None, None, np.ones(1, np.float32).ctypes.data, s) == 1


def test_body_generate_and_sharding(eng, six, ckpts):
    for e in (eng, six[0]):
        B, M = 6, 48
        mfcc = synth.synth_mfcc(B, M, seed=81)
        label = torch.arange(B) % 4
        seeds = _seeds(B, 81)
        pc = _per_clip(B)
        w = [SCALES[b % len(SCALES)] for b in range(B)]
        codes, poses, logp, glogp = (x.cpu() for x in e.body_generate(
            mfcc, label, None, seeds=seeds, want_logp=True, want_guide_logp=True, guidance=w,
            guide_mfcc=e.silence_mfcc(M, B), **pc))
        body = e.vq_decode(0, codes[..., 0].contiguous()).cpu()
        hand = e.vq_decode(1, codes[..., 1].contiguous()).cpu()
        assert torch.equal(poses, torch.cat([body, hand], 1).transpose(1, 2)), "poses decode the conditional codes"
        # the same pairs through pixelcnn_generate on the encoded audio
        aud = e.audio_encode(mfcc)
        sil = e.audio_encode(e.silence_mfcc(M, B))
        ref = e.pixelcnn_generate(aud, label, None, seeds=seeds, guidance=w, guide_aud=sil, **pc).cpu()
        assert torch.equal(codes, ref)
    e2 = _engine(ckpts["pixel"], ckpts["vq"])
    try:
        B, M = 10, 48
        mfcc = synth.synth_mfcc(B, M, seed=95)
        label = torch.arange(B) % 4
        seeds = _seeds(B, 95)
        pc = _per_clip(B)
        w = [SCALES[b % len(SCALES)] for b in range(B)]
        gl = (label + 1) % 4
        sl = lambda lo, hi: dict({k: v[lo:hi] for k, v in pc.items()}, guidance=w[lo:hi], guide_label=gl[lo:hi])
        c, p = (x.cpu() for x in eng.body_generate(mfcc, label, None, seeds=seeds, guidance=w, guide_label=gl, **pc))
        c0, p0 = (x.cpu() for x in eng.body_generate(mfcc[:4], label[:4], None, seeds=seeds[:4], **sl(0, 4)))
        c1, p1 = (x.cpu() for x in e2.body_generate(mfcc[4:], label[4:], None, seeds=seeds[4:], **sl(4, B)))
        assert torch.equal(torch.cat([c0, c1]), c) and torch.equal(torch.cat([p0, p1]), p)
    finally:
        torch.cuda.synchronize()
        e2.close()


def test_wholebody_generate(ckpts):
    """the overlapped WholeBody path forwards the guidance: its body codes are the engine's guided codes"""
    from talkshow_b200.engine import Engine, clip_seeds
    from talkshow_b200.pipeline import WholeBody

    wb = WholeBody(Engine(0))
    try:
        wb.load(ckpts["pixel"], ckpts["vq"], synth.face_checkpoint(0))
        B, M = 3, 40
        mfcc = synth.synth_mfcc(B, M, seed=7).cuda()
        wave = synth.synth_wave(B, 16000 * M // 30, seed=8).cuda()
        label = torch.arange(B).cuda()
        out = wb.generate(mfcc, wave, label, clip_seeds=5, guidance=2.0, guide_mfcc="silence", keep_logp=True,
                          keep_codes=True)
        torch.cuda.synchronize()
        assert out.shape[0] == B and torch.isfinite(out).all() and wb.last_guide_logp.shape == wb.last_logp.shape
        ref = wb.e.body_generate(mfcc, label, None, seeds=clip_seeds(5, B), guidance=2.0, guide_mfcc=wb.e.silence_mfcc(M, B))[0]
        assert torch.equal(wb.last_codes.cpu(), ref.cpu())
    finally:
        torch.cuda.synchronize()
        wb.close()
