"""CPU (-m "not gpu"): per-clip sampling controls of the body prior (each clip of a batch with its own temperature, top_k,
top_p and min_p).

tests/oracle_clip_ctl.py (the existing draws applied clip by clip) reproduces tests/golden/clip_ctl.npz, made by the
unmodified reference with its softmax swapped per batch row for the warp of that row's setting
(tests/golden/make_golden_clip_ctl.py).  The host layer (validation, forwarding, wrappers, WholeBody, sharded generation)
runs on the real library in host-only mode with its entry points recorded, and on an oracle-backed stand-in engine."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle_engine import OracleEngine
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_clip_ctl as OCC  # noqa: E402
import oracle_sampling as OSM  # noqa: E402
import oracle_style as OST  # noqa: E402

MIXED = [(0.8, 0, 1.0, 0.0), (0.0, 0, 1.0, 0.0), (1.0, 5, 0.9, 0.0), (1.3, 0, 1.0, 0.05)]


@pytest.fixture(scope="module")
def fix():
    return np.load(os.path.join(GOLDEN, "clip_ctl.npz"))


def _ckpts(key):
    if key == "6d":
        return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)
    return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0)


def test_fixture_is_the_checkpoints_and_is_unambiguous(fix):
    for key in ("3d", "6d"):
        ck, vq = _ckpts(key)
        assert np.allclose(fix["fp_%s" % key], list(synth.fingerprint(ck).values()))
        assert np.allclose(fix["fp_vq_%s" % key], list(synth.fingerprint(vq).values()))
        assert fix["codes_%s" % key].shape[0] == len(fix["settings"])
    s = fix["settings"]
    assert (s[:, 0] == 0).sum() >= 2 and (s[:, 2] < 1).any() and (s[:, 3] > 0).any() and (s[:, 1] > 0).any()
    assert float(fix["min_margin_top_p"]) >= 1e-5 and float(fix["min_margin_min_p"]) >= 1e-5


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_oracle_reproduces_reference(fix, key):
    torch.set_grad_enabled(False)
    ck, vq = _ckpts(key)
    settings = [tuple(r) for r in fix["settings"].tolist()]
    B = len(settings)
    mfcc = torch.from_numpy(fix["mfcc_%s" % key]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    noise = OSM.reference_noise(int(fix["seed_%s" % key]), 2 * T, B)
    label = torch.full((B,), int(fix["label_%s" % key]))
    style = OST.onehot(label, 4, T)
    codes, poses, logp, kept = OCC.body_sample(ck, vq, mfcc, style, noise, settings)
    assert torch.equal(codes, torch.from_numpy(fix["codes_%s" % key]))
    assert torch.equal(kept, torch.from_numpy(fix["kept_%s" % key]))
    assert (poses[:, ::int(fix["pose_stride"])] - torch.from_numpy(fix["poses_%s" % key])).abs().max() <= 1e-5
    assert (logp <= 0).all() and torch.isfinite(logp).all()
    # each clip equals its setting run alone (the per-clip rule is the scalar rule, clip by clip)
    for b in (0, 2, 4, B - 1):
        t, k, p, m = settings[b]
        one, _, _, kone = OST.body_sample(ck, vq, mfcc[b:b + 1], style[b:b + 1], noise[:, b:b + 1], t, int(k), p, m)
        assert torch.equal(one[0], codes[b]) and torch.equal(kone[0], kept[b]), b


def test_check_clip_controls():
    from talkshow_b200.engine import CLIP_CTL, check_clip_controls, per_clip, sampled

    cc = check_clip_controls([0.8, 0.0, 1.0], 5, np.array([1.0, 0.5, 0.9]), torch.tensor([0.0, 0.1, 0.0]))
    assert cc.dtype == CLIP_CTL and cc.shape == (3,)
    assert cc["temperature"].tolist() == [np.float32(0.8), 0.0, 1.0] and cc["top_k"].tolist() == [5, 5, 5]
    assert cc["min_p"][1] == np.float32(0.1)
    assert check_clip_controls(0.7, (0, 64), B=2)["top_k"].tolist() == [0, 64]
    assert not per_clip(0.7, 0, 1.0, 0.0) and not per_clip(torch.tensor(0.7), np.int64(3), np.float32(0.9), 0.0)
    assert per_clip(0.7, [3]) and per_clip(1.0, 0, torch.tensor([0.9]))
    assert sampled([0.0, 0.5]) and not sampled(np.zeros(3)) and sampled(0.1) and not sampled(0.0)
    bad = [
        (dict(temperature=[1.0, -0.5]), "clip 1"),
        (dict(temperature=[1.0, float("nan")]), "clip 1"),
        (dict(temperature=[1e39, 1.0]), "clip 0"),                   # finite in float64, inf in fp32
        (dict(top_k=[0, 2049]), "clip 1"),
        (dict(top_k=[2.5, 3]), "clip 0"),
        (dict(top_p=[0.9, 0.0]), "clip 1"),
        (dict(top_p=[1e-46, 0.9]), "clip 0"),                        # rounds to 0 in fp32
        (dict(min_p=[0.0, 1.5]), "clip 1"),
        (dict(top_k=[True, 3]), "clip 0"),
        (dict(temperature=np.array([True, False])), "clip 0"),
        (dict(temperature=[1.0, 1.0, 1.0]), "3 per-clip values for 2"),
        (dict(top_p=torch.ones(2, 1)), "one-dimensional"),
        (dict(temperature=[1.0, 1.0], top_k=-1), "top_k"),          # a bad broadcast scalar
        (dict(temperature=[1.0, "x"]), "clip 1"),
    ]
    for kw, msg in bad:
        args = dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            check_clip_controls(args["temperature"], args["top_k"], args["top_p"], args["min_p"], B=2)


class _RecordingLib:
    """stands in for the C library: records which entry point a call reaches with its arguments (a per-clip call's
    host controls copied out while the call runs) and returns success"""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name.startswith(("ts_pixelcnn_", "ts_body_")) and name not in ("ts_pixelcnn_row_bytes",):
            def call(*a):
                from talkshow_b200.engine import CLIP_CTL

                clip = None
                if name.endswith("_clips"):
                    nb = a[10]
                    clip = np.frombuffer(C.string_at(a[-2], nb * CLIP_CTL.itemsize), CLIP_CTL).copy()
                    ctl = a[-3]._obj
                    clip = (clip, (ctl.temperature, ctl.top_k, ctl.top_p, ctl.min_p), ctl.logp_out, ctl.kept_out)
                self.calls.append((name, a, clip))
                return 0
            return call
        return getattr(self.real, name)


def _recording_engine():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.load_pixelcnn(synth.pixelcnn_state(0))
    e.L = rec = _RecordingLib(e.L)
    e._s = lambda: None
    e.latent_rows = lambda M: M // 4
    e.vq_dim = lambda which: (39, 90)[which]
    return e, rec


def test_scalar_calls_forward_as_before():
    """all-scalar controls (Python, numpy or 0-d tensor scalars) reach the entry points they reached before: the per-clip
    path is taken only for per-clip values"""
    e, rec = _recording_engine()
    aud, label, mfcc = torch.zeros(2, 256, 5), torch.tensor([0, 1]), torch.zeros(2, 64, 20)
    noise, seeds = torch.ones(10, 2, 2048), torch.tensor([1, 2])
    anchors = torch.full((2, 5, 2), -1, dtype=torch.int64)
    style = torch.full((2, 5, 4), 0.25)
    cases = [(dict(), "generate"), (dict(temperature=0.7), "sample"), (dict(temperature=np.float32(0.7)), "sample"),
             (dict(temperature=torch.tensor(0.7), top_k=np.int64(5)), "sample"), (dict(top_p=0.9), "sample_ctl"),
             (dict(min_p=torch.tensor(0.05), want_logp=True), "sample_ctl"), (dict(seeds=seeds), "sample_seeded"),
             (dict(anchors=anchors, temperature=0.0), "sample_anchored"), (dict(style=style, top_k=3), "sample_styled")]
    for kw, want in cases:
        n = None if "seeds" in kw or kw.get("temperature") == 0.0 else noise
        e.pixelcnn_generate(aud, label, n, **kw)
        assert rec.calls[-1][0] == "ts_pixelcnn_" + want, kw
        e.body_generate(mfcc, label, n, **kw)
        assert rec.calls[-1][0] == "ts_body_" + want, kw
    e.close()


def test_per_clip_calls_reach_clip_entry_points():
    e, rec = _recording_engine()
    aud, label, mfcc = torch.zeros(4, 256, 5), torch.tensor([0, 1, 2, 3]), torch.zeros(4, 64, 20)
    noise, seeds = torch.ones(10, 4, 2048), torch.tensor([1, 2, 3, 4])
    t, k, p, m = (list(c) for c in zip(*MIXED))
    for call, name in ((lambda **kw: e.pixelcnn_generate(aud, label, **kw), "ts_pixelcnn_sample_clips"),
                       (lambda **kw: e.body_generate(mfcc, label, **kw), "ts_body_sample_clips")):
        call(noise=noise, temperature=t, top_k=k, top_p=p, min_p=m, want_logp=True, want_kept=True)
        got, a, (clip, ctl4, logp, kept) = rec.calls[-1]
        assert got == name
        assert [tuple(c) for c in clip.tolist()] == [tuple(np.float32(x).item() if i != 1 else x for i, x in enumerate(s))
                                                     for s in MIXED]
        assert logp and kept and a[4] == 4 and a[3].value is None      # no style: NULL, ncls unused
        # a scalar among per-clip values is broadcast; all-equal values still take the per-clip entry point
        call(noise=noise, temperature=np.full(4, 0.8, np.float32), top_k=64)
        got, a, (clip, _, logp, kept) = rec.calls[-1]
        assert got == name and clip["top_k"].tolist() == [64] * 4 and logp is None and kept is None
        assert np.all(clip["temperature"] == np.float32(0.8))
        # seeds, anchors and style ride along; a batch of greedy clips needs neither noise nor seeds
        call(noise=None, seeds=seeds, temperature=torch.tensor([0.5, 0.0, 1.0, 2.0]), style=torch.full((4, 5, 4), 0.25),
             anchors=torch.full((4, 5, 2), -1, dtype=torch.int64))
        got, a, _ = rec.calls[-1]
        assert got == name and a[3].value is not None and a[6].value is not None and a[7].value is not None
        call(noise=None, temperature=[0.0, 0.0, 0.0, 0.0], top_k=[1, 2, 3, 4])
        assert rec.calls[-1][0] == name and rec.calls[-1][1][5].value is None and rec.calls[-1][1][6].value is None
    n = len(rec.calls)
    for kw in (dict(noise=None, temperature=[0.0, 0.5, 0.0, 0.0]),                    # a sampled clip without a source
               dict(noise=noise, seeds=seeds, temperature=[0.0, 0.5, 0.0, 0.0]),     # two sources
               dict(noise=noise, temperature=[1.0, 1.0, 1.0]),                        # wrong length
               dict(noise=noise, top_k=[0, 0, True, 0]),                              # a bool
               dict(noise=noise, top_p=[0.9, 0.9, 1.2, 0.9]),                         # out of range
               dict(noise=noise, min_p=torch.zeros(4, 1))):                           # not 1-D
        with pytest.raises(ValueError):
            e.pixelcnn_generate(aud, label, **kw)
        with pytest.raises(ValueError):
            e.body_generate(mfcc, label, **kw)
    assert len(rec.calls) == n                                                       # rejected before any call
    with pytest.raises(ValueError, match="clip 2"):
        e.pixelcnn_generate(aud, label, noise, top_p=[0.9, 0.9, 1.2, 0.9])
    e.close()


def test_per_clip_chunks_slice_the_controls():
    """a batch above the 64-sample tile: one call per chunk, each with its clips' controls"""
    e, rec = _recording_engine()
    B = 100
    t = np.linspace(0.0, 1.5, B)
    k = np.arange(B) % 7
    e.pixelcnn_generate(torch.zeros(B, 256, 5), torch.tensor([0]), torch.ones(10, B, 2048), temperature=t, top_k=k)
    e.body_generate(torch.zeros(B, 64, 20), torch.tensor([1]), torch.ones(10, B, 2048), temperature=t, top_k=k)
    assert [c[0] for c in rec.calls] == ["ts_pixelcnn_sample_clips"] * 2 + ["ts_body_sample_clips"] * 2
    for i in (0, 2):
        clips = np.concatenate([rec.calls[i][2][0], rec.calls[i + 1][2][0]])
        assert [c[1][10] for c in rec.calls[i:i + 2]] == [64, 36]
        assert np.array_equal(clips["temperature"], t.astype(np.float32)) and np.array_equal(clips["top_k"], k)
    e.close()


class ClipOracleEngine(OracleEngine):
    """OracleEngine whose sampling calls take the controls (scalar or per clip), ``seeds=``-free noise, ``anchors=`` and
    ``style=`` of Engine and are answered by tests/oracle_clip_ctl.py.  Every call is recorded in ``calls`` as (method,
    CLIP_CTL array)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    def load_pixelcnn(self, sd):
        super().load_pixelcnn(sd)
        self.pixelcnn_ncls = sd["layers.0.class_cond_embedding.weight"].shape[0]

    def _prep(self, name, B, H, label, style, temperature, top_k, top_p, min_p, noise):
        from talkshow_b200.engine import check_clip_controls, check_style

        clip = check_clip_controls(temperature, top_k, top_p, min_p, B)
        self.calls.append((name, clip))
        if style is not None:
            st = check_style(style, B, H, self.pixelcnn_ncls)
        else:
            label = label.reshape(-1).to(torch.int64)
            st = OST.onehot(label.expand(B) if label.numel() == 1 else label, self.pixelcnn_ncls, H)
        assert noise is not None or not (clip["temperature"] > 0).any()
        return clip, st

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, temperature=1.0, top_k=0,
                          want_logp=False, top_p=1.0, min_p=0.0, want_kept=False, anchors=None, style=None):
        B = aud.shape[0]
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        T = aud.shape[2] - T0 if T is None else T
        clip, st = self._prep("pixelcnn_generate", B, T0 + T, label, style, temperature, top_k, top_p, min_p, noise)
        a2 = aud.float().unsqueeze(-1).repeat(1, 1, 1, 2)
        pre = dict(pre_latents=pre_latents, pre_audio=a2[:, :, :T0]) if T0 else {}
        codes, logp, kept = OCC.pixelcnn_sample(self.sd["pixelcnn"], st, T, B, a2[:, :, T0:], noise, clip, anchors=anchors,
                                                window=self.window, **pre)
        out = (codes,) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())
        return out if len(out) > 1 else codes

    def body_generate(self, mfcc, label, noise, want_codes=True, temperature=1.0, top_k=0, want_logp=False, top_p=1.0,
                      min_p=0.0, want_kept=False, anchors=None, style=None):
        B, T = mfcc.shape[0], self.latent_rows(mfcc.shape[2])
        clip, st = self._prep("body_generate", B, T, label, style, temperature, top_k, top_p, min_p, noise)
        codes, poses, logp, kept = OCC.body_sample({"generator": self.sd["pixelcnn"], "audioencoder": self.sd["audioenc"]},
                                                   {"g_body": self.sd["vq0"], "g_hand": self.sd["vq1"]}, mfcc.float(), st,
                                                   noise, clip, anchors=anchors, window=self.window)
        return ((codes if want_codes else None), poses) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())


def _wrapper(engine):
    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Model.vq_path = ""
    g = TrainWrapper(types.SimpleNamespace(gpu=0, infer=True), cfg, engine=engine)
    ck, vq = _ckpts("3d")
    g.load_state_dict(ck)
    g.load_vq_state_dict(vq)
    return g


def _controls(clip):
    return [c.tolist() for c in (clip["temperature"], clip["top_k"], clip["top_p"], clip["min_p"])]


def test_wrappers_forward_per_clip_controls(monkeypatch):
    from talkshow_b200.nets import smplx_body_pixel as bp

    torch.set_grad_enabled(False)
    e = ClipOracleEngine()
    g = _wrapper(e)
    g.noise_device = "cpu"
    B, M = 4, 16
    mfcc = synth.synth_mfcc(B, M, seed=14)
    label = torch.tensor([0, 1, 2, 3])
    t, k, p, m = (list(c) for c in zip(*MIXED))
    want = _controls(np.array(MIXED, dtype=[(n, d) for n, d in zip(("temperature", "top_k", "top_p", "min_p"),
                                                                    ("<f4", "<i4", "<f4", "<f4"))]))
    noise = OSM.reference_noise(15, 2 * (M // 4), B)
    g.generate(mfcc, label, noise_fn=lambda T_, B_: noise, temperature=t, top_k=k, top_p=p, min_p=m, keep_logp=True)
    assert _controls(e.calls[-1][1]) == want and g.last_kept is not None and g.last_logp is not None
    per_clip_codes = g.last_codes
    for b in range(B):          # each clip equals its setting run alone (the scalar path of the same stand-in)
        g.generate(mfcc[b:b + 1], label[b:b + 1], noise_fn=lambda T_, B_: noise[:, b:b + 1], temperature=t[b], top_k=k[b],
                   top_p=p[b], min_p=m[b])
        assert torch.equal(g.last_codes[0], per_clip_codes[b]), b
    feat = mfcc.transpose(1, 2)
    lat0, a0, _, _ = g.infer(feat, 0, label, B, noise_fn=lambda T_, B_: noise, temperature=t)
    assert _controls(e.calls[-1][1])[0] == want[0]
    g.infer(feat, 0, label, B, lat0, a0, noise_fn=lambda T_, B_: noise, top_k=k)
    assert _controls(e.calls[-1][1])[1] == k
    # greedy clips everywhere: no noise is drawn
    g.noise_fn_calls = 0
    g.generate(mfcc, label, noise_fn=lambda T_, B_: pytest.fail("noise drawn for greedy clips"), temperature=[0.0] * B)
    g.infer_on_audio(mfcc[0].transpose(0, 1).numpy(), B=B, temperature=t, top_p=p)
    assert _controls(e.calls[-1][1])[2] == want[2]
    # continuity: both chunks take each clip's setting
    monkeypatch.setattr(bp, "get_mfcc_sepa", lambda *a, **kk: (np.asarray(synth.synth_mfcc(1, 40, seed=5)[0].T), 16))
    n = len(e.calls)
    g.infer_on_audio("unused.wav", B=B, continuity=True, temperature=t, min_p=m, clip_seeds=None)
    assert len(e.calls) == n + 2
    for _, clip in e.calls[-2:]:
        assert _controls(clip)[0] == want[0] and _controls(clip)[3] == want[3]
    for bad in (dict(temperature=t[:3]), dict(top_k=[0, 1, True, 3]), dict(top_p=[0.9, 0.0, 1.0, 1.0])):
        with pytest.raises(ValueError):
            g.generate(mfcc, label, **bad)


def test_wholebody_and_sharded_with_per_clip_controls():
    from talkshow_b200.pipeline import WholeBody, shard_range

    torch.set_grad_enabled(False)
    e = ClipOracleEngine()
    wb = WholeBody(e)
    wb.load(synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), synth.face_checkpoint(0))
    B, M = 5, 16
    T = M // 4
    mfcc = synth.synth_mfcc(B, M, seed=36)
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(37))
    label = torch.tensor([0, 1, 3, 2, 0])
    t = [0.8, 0.0, 1.0, 1.3, 0.0]
    k = np.array([0, 0, 5, 0, 3])
    p = torch.tensor([1.0, 1.0, 0.9, 1.0, 1.0])
    noise = OSM.reference_noise(39, 2 * T, B)
    one = wb.generate(mfcc, wave, label, noise=noise, temperature=t, top_k=k, top_p=p, min_p=0.0, keep_logp=True,
                      keep_codes=True)
    full = e.calls[-1][1]
    assert _controls(full)[1] == k.tolist() and wb.last_kept is not None
    codes = wb.last_codes
    for b in (1, 2):
        wb.generate(mfcc[b:b + 1], wave[b:b + 1], label[b:b + 1], noise=noise[:, b:b + 1], temperature=t[b], top_k=int(k[b]),
                    top_p=float(p[b]), keep_codes=True)
        assert torch.equal(wb.last_codes[0], codes[b]), b
    for world in (1, 2, 3):
        parts = []
        for r in range(world):
            parts.append(wb.generate_sharded(mfcc, wave, label, r, world, noise_full=noise, gather=False, temperature=t,
                                             top_k=k, top_p=p))
            lo, hi = shard_range(B, r, world)
            assert np.array_equal(e.calls[-1][1], full[lo:hi]), (world, r)     # rank r passes its shard's controls
        # the CPU stand-in's modules round differently at different batch sizes; the GPU test compares bit for bit
        assert (torch.cat(parts) - one).abs().max() <= 1e-5, world
    with pytest.raises(ValueError):
        wb.generate_sharded(mfcc, wave, label, 0, 2, noise_full=noise, temperature=t[:4])
