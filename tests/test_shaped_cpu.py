"""CPU (-m "not gpu"): logit shaping of the body prior (a repetition penalty over each clip's recent codes and an additive
code bias).

tests/oracle_shaped.py reproduces tests/golden/shaped.npz, made by the unmodified reference with its softmax swapped per
batch row for the shaping and the warp of that row's setting (tests/golden/make_golden_shaped.py).  The host layer
(validation, forwarding, chunking, wrappers, WholeBody, sharded generation) runs on the real library in host-only mode
with its entry points recorded, and on the oracle-backed stand-in engine of oracle_shaped."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_sampling as OSM  # noqa: E402
import oracle_shaped as OSH  # noqa: E402
import oracle_style as OST  # noqa: E402
import talkshow_oracle as O  # noqa: E402
from test_clip_ctl_cpu import _RecordingLib, _wrapper  # noqa: E402


@pytest.fixture(scope="module")
def fix():
    return np.load(os.path.join(GOLDEN, "shaped.npz"))


def _ckpts(six):
    if six:
        return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)
    return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0)


def _settings(fix):
    s = fix["settings"].tolist()
    return [tuple(r[:4]) for r in s], [(r[4], int(r[5])) for r in s]


def test_fixture_is_the_checkpoints_and_is_unambiguous(fix):
    for case, six in (("3d", False), ("pre", False), ("6d", True)):
        ck, vq = _ckpts(six)
        assert np.allclose(fix["fp_%s" % case], list(synth.fingerprint(ck).values()))
        assert np.allclose(fix["fp_vq_%s" % case], list(synth.fingerprint(vq).values()))
        bias = fix["bias_%s" % case]
        assert (np.isfinite(bias).any(-1)).all() and (np.abs(bias[np.isfinite(bias)]) <= 1e4).all()
        assert (bias == -np.inf).any() and (fix["kept_%s" % case] >= 1).all()
    assert float(fix["min_margin_top_p"]) >= 1e-5 and float(fix["min_margin_min_p"]) >= 1e-5
    # the prefix case's windows reach into the prefix, which repeats its last codes
    pre = fix["pre_pre"]
    assert (pre[:, -1] == pre[:, -2]).all()


@pytest.mark.parametrize("case", ["3d", "pre", "6d"])
def test_oracle_reproduces_reference(fix, case):
    torch.set_grad_enabled(False)
    ck, vq = _ckpts(case == "6d")
    clip, shapes = _settings(fix)
    B = len(clip)
    mfcc = torch.from_numpy(fix["mfcc_%s" % case]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    noise = OSM.reference_noise(int(fix["seed_%s" % case]), 2 * T, B)
    label = torch.full((B,), int(fix["label_%s" % case]))
    bias = torch.from_numpy(fix["bias_%s" % case])
    if case == "pre":
        pre = torch.from_numpy(fix["pre_pre"])
        T0 = pre.shape[1]
        a = O.audio_encoder(ck["audioencoder"], mfcc).unsqueeze(-1).repeat(1, 1, 1, 2)
        ap = O.audio_encoder(ck["audioencoder"], torch.from_numpy(fix["mfcc_pre_pre"]).repeat(B, 1, 1))
        ap = ap.unsqueeze(-1).repeat(1, 1, 1, 2)
        style = OST.onehot(label, 4, T0 + T)
        codes, logp, kept = OSH.pixelcnn_sample(ck["generator"], style, T, B, a, noise, clip, shapes, bias=bias,
                                                pre_latents=pre, pre_audio=ap)
    else:
        style = OST.onehot(label, 4, T)
        codes, poses, logp, kept = OSH.body_sample(ck, vq, mfcc, style, noise, clip, shapes, bias=bias)
        assert (poses[:, ::int(fix["pose_stride"])] - torch.from_numpy(fix["poses_%s" % case])).abs().max() <= 1e-5
    assert torch.equal(codes, torch.from_numpy(fix["codes_%s" % case]))
    assert torch.equal(kept, torch.from_numpy(fix["kept_%s" % case]))
    assert (logp <= 0).all() and torch.isfinite(logp).all()
    assert not (bias.gather(-1, codes.transpose(1, 2)) == float("-inf")).any()


def test_shaping_changes_the_draw():
    """the penalty and the bias act: the greedy loop of a prior is broken, and a banned code is never drawn"""
    l = torch.tensor([3.0, -1.0, 2.5, 0.5])
    s = OSH.shape(l, torch.tensor([0, 0, 1]), 2.0)
    assert s.tolist() == [1.5, -2.0, 2.5, 0.5]
    assert OSH.shape(l, torch.tensor([0]), 1.0, torch.tensor([0.0, 0.0, float("-inf"), 1.0])).tolist() == \
        [3.0, -1.0, float("-inf"), 1.5]
    lg = torch.randn(1, 2048, generator=torch.Generator().manual_seed(1))
    lg[0, 7] = float("-inf")
    code, kept = OSH.draw(lg, torch.ones(1, 2048), 1.0, 2048)
    assert kept.item() == 2047 and code.item() != 7
    _, kept = OSH.draw(lg, torch.ones(1, 2048), 1.0, 5)
    assert kept.item() == 5


def test_check_clip_shape_and_code_bias():
    from talkshow_b200.engine import CLIP_SHAPE, check_clip_shape, check_code_bias, shaping_kwargs

    cs = check_clip_shape([1.0, 1.5, np.float32(2.0)], 4, B=3)
    assert cs.dtype == CLIP_SHAPE and cs["repetition_penalty"].tolist() == [1.0, 1.5, 2.0]
    assert cs["repetition_window"].tolist() == [4, 4, 4]
    assert check_clip_shape(1.3, torch.tensor([1, 8]))["repetition_window"].tolist() == [1, 8]
    bad = [
        (dict(repetition_penalty=0.9), "repetition_penalty"),
        (dict(repetition_penalty=[1.0, 0.5]), "clip 1"),
        (dict(repetition_penalty=[float("nan"), 1.0]), "clip 0"),
        (dict(repetition_penalty=[1.0, float("inf")]), "clip 1"),
        (dict(repetition_penalty=[1.0, 1e39]), "clip 1"),                  # finite in float64, inf in fp32
        (dict(repetition_penalty=[True, 1.0]), "clip 0"),
        (dict(repetition_penalty=True), "repetition_penalty"),
        (dict(repetition_penalty="x"), "repetition_penalty"),
        (dict(repetition_window=[8, 0]), "clip 1"),
        (dict(repetition_window=[8, 2.5]), "clip 1"),
        (dict(repetition_window=[False, 8]), "clip 0"),
        (dict(repetition_window=2 ** 31), "repetition_window"),
        (dict(repetition_window=[8, 8, 8]), "3 per-clip values for 2"),
        (dict(repetition_penalty=torch.ones(2, 1)), "one-dimensional"),
    ]
    for kw, msg in bad:
        args = dict(repetition_penalty=1.0, repetition_window=8)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            check_clip_shape(args["repetition_penalty"], args["repetition_window"], B=2)
    b = np.zeros((2, 2048), np.float64)
    b[0, :5] = -np.inf
    got = check_code_bias(b, 3)
    assert got.dtype == torch.float32 and got.shape == (3, 2, 2048) and got.is_contiguous()
    assert torch.isinf(got[2, 0, :5]).all()
    assert check_code_bias(torch.ones(3, 2, 2048, dtype=torch.int32), 3).dtype == torch.float32
    for val, where in ((float("inf"), "clip 1, column 0"), (float("nan"), "clip 2, column 1"), (2e4, "clip 1, column 0")):
        bb = torch.zeros(3, 2, 2048)
        c = 0 if "column 0" in where else 1
        bb[int(where[5]), c, 9] = val
        with pytest.raises(ValueError, match=where):
            check_code_bias(bb, 3)
    bb = torch.zeros(3, 2, 2048)
    bb[1, 1] = float("-inf")
    with pytest.raises(ValueError, match="clip 1, column 1 .hand.: every code is -inf"):
        check_code_bias(bb, 3)
    for x, msg in ((torch.zeros(3, 2, 2047), "shape"), (torch.zeros(2, 2, 2048), "shape"), ([0.0] * 2048, "tensor"),
                   (np.zeros((2, 2048), bool), "dtype"), (torch.zeros(2, 2048, dtype=torch.bool), "float")):
        with pytest.raises(ValueError, match=msg):
            check_code_bias(x, 3)
    assert shaping_kwargs(1.0, 8, None, 2) == {} and shaping_kwargs([1.0, 1.0], 3, None, 2) == {}
    assert set(shaping_kwargs(1.2, 8, None, 2)) == {"repetition_penalty", "repetition_window", "code_bias"}
    assert shaping_kwargs(1.0, 8, torch.zeros(2, 2048), 2)["code_bias"] is not None
    with pytest.raises(ValueError):
        shaping_kwargs(1.0, 0, None, 2)                                      # the window is checked even when off


class _ShapeRecordingLib(_RecordingLib):
    """_RecordingLib that also copies out a shaped call's host shaping entries"""

    def __getattr__(self, name):
        f = super().__getattr__(name)
        if not name.endswith("_shaped"):
            return f

        def call(*a):
            from talkshow_b200.engine import CLIP_CTL, CLIP_SHAPE

            nb = a[10]
            clip = None if a[-4] is None else np.frombuffer(C.string_at(a[-4], nb * CLIP_CTL.itemsize), CLIP_CTL).copy()
            shape = None if a[-3] is None else np.frombuffer(C.string_at(a[-3], nb * CLIP_SHAPE.itemsize), CLIP_SHAPE).copy()
            ctl = a[-5]._obj
            self.calls.append((name, a, (clip, shape, a[-2].value, (ctl.temperature, ctl.top_k, ctl.top_p, ctl.min_p))))
            return 0
        return call


def _recording_engine():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.load_pixelcnn(synth.pixelcnn_state(0))
    e.L = rec = _ShapeRecordingLib(e.L)
    e._s = lambda: None
    e.latent_rows = lambda M: M // 4
    e.vq_dim = lambda which: (39, 90)[which]
    return e, rec


def test_calls_without_shaping_forward_as_before():
    """no shaping keyword, theta 1 (scalar or per clip) with any window: the entry points the call reached before"""
    e, rec = _recording_engine()
    aud, label, mfcc = torch.zeros(2, 256, 5), torch.tensor([0, 1]), torch.zeros(2, 64, 20)
    noise = torch.ones(10, 2, 2048)
    cases = [(dict(), "generate"), (dict(temperature=0.7), "sample"), (dict(top_p=0.9), "sample_ctl"),
             (dict(temperature=[0.7, 0.0]), "sample_clips"), (dict(repetition_penalty=1.0, repetition_window=3), "generate"),
             (dict(repetition_penalty=[1.0, 1.0], temperature=0.7), "sample")]
    for kw, want in cases:
        e.pixelcnn_generate(aud, label, noise, **kw)
        assert rec.calls[-1][0] == "ts_pixelcnn_" + want, kw
        e.body_generate(mfcc, label, noise, **kw)
        assert rec.calls[-1][0] == "ts_body_" + want, kw
    e.close()


def test_shaped_calls_reach_shaped_entry_points():
    e, rec = _recording_engine()
    aud, label, mfcc = torch.zeros(3, 256, 5), torch.tensor([0, 1, 2]), torch.zeros(3, 64, 20)
    noise = torch.ones(10, 3, 2048)
    bias = torch.zeros(2, 2048)
    bias[1, 3] = float("-inf")
    for call, name in ((lambda **kw: e.pixelcnn_generate(aud, label, **kw), "ts_pixelcnn_sample_shaped"),
                       (lambda **kw: e.body_generate(mfcc, label, **kw), "ts_body_sample_shaped")):
        call(noise=noise, repetition_penalty=1.5, temperature=0.8, top_k=5)
        got, a, (clip, shape, bptr, ctl4) = rec.calls[-1]
        assert got == name and clip is None and bptr is None and ctl4 == (np.float32(0.8), 5, 1.0, 0.0)
        assert shape["repetition_penalty"].tolist() == [1.5] * 3 and shape["repetition_window"].tolist() == [8] * 3
        call(noise=noise, repetition_penalty=[1.0, 2.0, 1.0], repetition_window=[1, 2, 3], temperature=[0.5, 0.0, 1.0])
        got, a, (clip, shape, bptr, _) = rec.calls[-1]
        assert got == name and clip["temperature"].tolist() == [0.5, 0.0, 1.0]
        assert shape["repetition_penalty"].tolist() == [1.0, 2.0, 1.0] and shape["repetition_window"].tolist() == [1, 2, 3]
        call(noise=None, temperature=0.0, code_bias=bias)                # a bias alone: no penalty entries
        got, a, (clip, shape, bptr, _) = rec.calls[-1]
        assert got == name and shape is None and bptr
    n = len(rec.calls)
    bad_bias = torch.zeros(3, 2, 2048)
    bad_bias[2, 0] = float("-inf")
    for kw in (dict(noise=noise, repetition_penalty=0.5), dict(noise=noise, repetition_window=[1, 2]),
               dict(noise=noise, code_bias=bad_bias), dict(noise=noise, code_bias=torch.zeros(4, 2, 2048)),
               dict(noise=None, repetition_penalty=2.0)):
        with pytest.raises(ValueError):
            e.pixelcnn_generate(aud, label, **kw)
        with pytest.raises(ValueError):
            e.body_generate(mfcc, label, **kw)
    assert len(rec.calls) == n                                          # rejected before any call
    e.close()


def test_chunks_slice_the_shaping():
    """a batch above the 64-sample tile: one call per chunk, each with its clips' penalties, windows and bias rows"""
    e, rec = _recording_engine()
    B = 100
    th = np.linspace(1.0, 3.0, B)
    w = np.arange(B) % 9 + 1
    bias = torch.randn(B, 2, 2048)
    e.pixelcnn_generate(torch.zeros(B, 256, 5), torch.tensor([0]), torch.ones(10, B, 2048), repetition_penalty=th,
                        repetition_window=w, code_bias=bias)
    e.body_generate(torch.zeros(B, 64, 20), torch.tensor([1]), torch.ones(10, B, 2048), repetition_penalty=th,
                    repetition_window=w, code_bias=bias)
    assert [c[0] for c in rec.calls] == ["ts_pixelcnn_sample_shaped"] * 2 + ["ts_body_sample_shaped"] * 2
    for i in (0, 2):
        shape = np.concatenate([rec.calls[i][2][1], rec.calls[i + 1][2][1]])
        assert [c[1][10] for c in rec.calls[i:i + 2]] == [64, 36]
        assert np.array_equal(shape["repetition_penalty"], th.astype(np.float32))
        assert np.array_equal(shape["repetition_window"], w)
        assert rec.calls[i + 1][2][2] - rec.calls[i][2][2] == 64 * 2 * 2048 * 4       # the bias rows of the second chunk
    e.close()


def _last(e):
    name, clip, shape, bias = e.calls[-1]
    return shape["repetition_penalty"].tolist(), shape["repetition_window"].tolist(), bias


def test_wrappers_forward_the_shaping(monkeypatch):
    from talkshow_b200.nets import smplx_body_pixel as bp

    torch.set_grad_enabled(False)
    e = OSH.ShapedOracleEngine()
    g = _wrapper(e)
    g.noise_device = "cpu"
    B, M = 3, 16
    mfcc = synth.synth_mfcc(B, M, seed=24)
    label = torch.tensor([0, 1, 2])
    noise = OSM.reference_noise(25, 2 * (M // 4), B)
    th, w = [1.0, 2.0, 3.0], [1, 4, 8]
    bias = torch.zeros(B, 2, 2048)
    bias[:, :, :1000] = float("-inf")
    g.generate(mfcc, label, noise_fn=lambda T_, B_: noise, temperature=0.0, repetition_penalty=th, repetition_window=w,
               code_bias=bias, keep_logp=True)
    assert _last(e)[:2] == (th, w) and torch.equal(_last(e)[2], bias)
    assert (g.last_codes >= 1000).all()
    greedy = g.last_codes
    for b in range(B):          # each clip equals its setting run alone
        g.generate(mfcc[b:b + 1], label[b:b + 1], temperature=0.0, repetition_penalty=th[b], repetition_window=w[b],
                   code_bias=bias[b])
        assert torch.equal(g.last_codes[0], greedy[b]), b
    # the penalty breaks greedy repetition: with theta 3 over the whole history no code repeats as often
    g.generate(mfcc, label, temperature=0.0)
    plain = g.last_codes
    g.generate(mfcc, label, temperature=0.0, repetition_penalty=100.0, repetition_window=1000)
    rep = lambda c: int((c[:, 1:] == c[:, :-1]).sum())
    assert rep(g.last_codes) <= rep(plain)
    n = len(e.calls)
    g.generate(mfcc, label, temperature=0.0)
    assert _last(e)[:2] == ([1.0] * B, [8] * B) and _last(e)[2] is None and len(e.calls) == n + 1
    feat = mfcc.transpose(1, 2)
    lat0, a0, _, _ = g.infer(feat, 0, label, B, noise_fn=lambda T_, B_: noise, repetition_penalty=1.5)
    assert _last(e)[0] == [1.5] * B
    g.infer(feat, 0, label, B, lat0, a0, noise_fn=lambda T_, B_: noise, code_bias=bias[0])
    assert torch.equal(_last(e)[2], bias)
    g.infer_on_audio(mfcc[0].transpose(0, 1).numpy(), B=B, temperature=0.0, repetition_penalty=th, repetition_window=w)
    assert _last(e)[:2] == (th, w)
    # continuity: both chunks take each clip's shaping; chunk 1's window reaches into chunk 0's codes (pre_latents)
    monkeypatch.setattr(bp, "get_mfcc_sepa", lambda *a, **kk: (np.asarray(synth.synth_mfcc(1, 40, seed=5)[0].T), 16))
    n = len(e.calls)
    g.infer_on_audio("unused.wav", B=B, continuity=True, temperature=0.0, repetition_penalty=th, repetition_window=w,
                     code_bias=bias)
    assert len(e.calls) == n + 2
    for _, clip, shape, bb in e.calls[-2:]:
        assert shape["repetition_penalty"].tolist() == th and torch.equal(bb, bias)
    for bad in (dict(repetition_penalty=th[:2]), dict(repetition_window=[1, 0, 2]), dict(code_bias=torch.zeros(2, 2, 2048))):
        with pytest.raises(ValueError):
            g.generate(mfcc, label, **bad)


def test_wholebody_and_sharded_with_shaping():
    from talkshow_b200.pipeline import WholeBody, shard_range

    torch.set_grad_enabled(False)
    e = OSH.ShapedOracleEngine()
    wb = WholeBody(e)
    wb.load(synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), synth.face_checkpoint(0))
    B, M = 5, 16
    T = M // 4
    mfcc = synth.synth_mfcc(B, M, seed=36)
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(37))
    label = torch.tensor([0, 1, 3, 2, 0])
    th = [1.0, 1.5, 2.0, 3.0, 1.2]
    w = np.array([8, 1, 4, 100, 2])
    bias = torch.randn(B, 2, 2048, generator=torch.Generator().manual_seed(38))
    bias[:, :, ::3] = float("-inf")
    noise = OSM.reference_noise(39, 2 * T, B)
    one = wb.generate(mfcc, wave, label, noise=noise, repetition_penalty=th, repetition_window=w, code_bias=bias,
                      keep_codes=True)
    full = e.calls[-1]
    assert full[2]["repetition_window"].tolist() == w.tolist() and torch.equal(full[3], bias)
    assert not (wb.last_codes % 3 == 0).any()
    for world in (1, 2, 3):
        parts = []
        for r in range(world):
            parts.append(wb.generate_sharded(mfcc, wave, label, r, world, noise_full=noise, gather=False,
                                             repetition_penalty=th, repetition_window=w, code_bias=bias))
            lo, hi = shard_range(B, r, world)
            assert np.array_equal(e.calls[-1][2], full[2][lo:hi]), (world, r)      # rank r passes its shard's values
            assert torch.equal(e.calls[-1][3], bias[lo:hi]), (world, r)
        assert (torch.cat(parts) - one).abs().max() <= 1e-5, world
    n = len(e.calls)
    wb.generate_sharded(mfcc, wave, label, 0, 2, noise_full=noise, gather=False)
    assert e.calls[-1][3] is None and e.calls[-1][2]["repetition_penalty"].tolist() == [1.0] * 3 and len(e.calls) == n + 1
    with pytest.raises(ValueError):
        wb.generate_sharded(mfcc, wave, label, 0, 2, noise_full=noise, repetition_penalty=th[:4])
