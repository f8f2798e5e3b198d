"""CPU (-m "not gpu"): guided sampling of the body prior (ts_pixelcnn_sample_guided / ts_body_sample_guided).

The oracle (tests/oracle_guided.py) is checked against the shaped oracle at w = 1 and against the rule's fp32 arithmetic.
The host layer (validation, interleaving of the two branches, per-pair draw inputs, 32-pair chunks, the wrappers and
WholeBody) runs on the real library in host-only mode with its entry points recorded."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_guided as OG  # noqa: E402
import oracle_sampling as OSM  # noqa: E402
import oracle_shaped as OSH  # noqa: E402
import oracle_style as OST  # noqa: E402
import talkshow_oracle as O  # noqa: E402
from test_clip_ctl_cpu import _RecordingLib, _recording_engine  # noqa: E402


def _i64(ptr, n):
    return np.frombuffer(C.string_at(ptr, 8 * n), np.int64).copy()


def _f32(ptr, n):
    return np.frombuffer(C.string_at(ptr, 4 * n), np.float32).copy()


class _GuidedRecordingLib(_RecordingLib):
    """_RecordingLib that also copies out what a guided call passes: the branch labels, the pair scales and the per-pair
    controls (host memory, read while the call runs)."""

    def __getattr__(self, name):
        if name in ("ts_pixelcnn_sample_guided", "ts_body_sample_guided"):
            from talkshow_b200.engine import CLIP_CTL, CLIP_SHAPE

            def call(*a):
                P = a[10]
                ctl = a[-6]._obj
                a = tuple(x.value if isinstance(x, C.c_void_p) else x for x in a)
                rec = dict(P=P, label=None if not a[2] else _i64(a[2], 2 * P), style=a[3], noise=a[5], seeds=a[6],
                           anchors=a[7], guidance=_f32(a[-2], P), ctl=(ctl.temperature, ctl.top_k, ctl.top_p, ctl.min_p),
                           clip=None if not a[-5] else np.frombuffer(C.string_at(a[-5], P * CLIP_CTL.itemsize), CLIP_CTL).copy(),
                           shape=None if not a[-4] else np.frombuffer(C.string_at(a[-4], P * CLIP_SHAPE.itemsize),
                                                                      CLIP_SHAPE).copy(), bias=a[-3])
                if a[3] and name == "ts_pixelcnn_sample_guided":   # the branch schedules [2P][T0+T][4]
                    rec["style_rows"] = _f32(a[3], 2 * P * (a[11] + a[13]) * 4).reshape(2 * P, a[11] + a[13], 4)
                self.calls.append((name, a, rec))
                return 0
            return call
        return super().__getattr__(name)


def _engine():
    e, rec = _recording_engine()
    e.L = rec = _GuidedRecordingLib(rec.real)
    return e, rec


def test_guided_logits_arithmetic():
    """three separately rounded fp32 operations; w = 1 returns l_c"""
    g = torch.Generator().manual_seed(1)
    lc, lu = torch.randn(2048, generator=g) * 5, torch.randn(2048, generator=g) * 5
    assert torch.equal(OG.guided_logits(lc, lu, 1.0), lc)
    for w in (0.0, 0.5, 1.5, 2.0, 3.0, 100.0):
        s = np.float32(w) - np.float32(1)
        d = (lc.numpy() - lu.numpy()).astype(np.float32)
        want = (lc.numpy() + (s * d).astype(np.float32)).astype(np.float32)
        assert np.array_equal(OG.guided_logits(lc, lu, w).numpy(), want)
    assert (OG.guided_logits(lc, lu, 0.0) - lu).abs().max() <= 1e-5   # w = 0: the negative branch's logits, up to rounding


def test_oracle_identity_and_effect():
    """w = 1: the pair draws what the shaped oracle draws on the conditional branch; w != 1 against a different negative
    audio changes the draws"""
    torch.set_grad_enabled(False)
    ck = synth.body_pixel_checkpoint(0)
    P, T = 3, 6
    aud = O.audio_encoder(ck["audioencoder"], synth.synth_mfcc(P, 4 * T, seed=5)).unsqueeze(-1).repeat(1, 1, 1, 2)
    neg = O.audio_encoder(ck["audioencoder"], synth.synth_mfcc(P, 4 * T, seed=6)).unsqueeze(-1).repeat(1, 1, 1, 2)
    label = torch.tensor([0, 1, 2])
    style = OST.onehot(label, 4, T)
    style2 = torch.stack([style, style], 1).reshape(2 * P, T, 4)
    aud2 = torch.stack([aud, neg], 1).reshape((2 * P,) + tuple(aud.shape[1:]))
    noise = OSM.reference_noise(3, 2 * T, P)
    clip = [(0.8, 0, 1.0, 0.0), (0.0, 0, 1.0, 0.0), (1.0, 64, 1.0, 0.0)]
    shapes = [(1.0, 8), (1.5, 2), (1.0, 8)]
    codes, logp, kept = OG.pixelcnn_sample(ck["generator"], style2, T, P, aud2, noise, clip, shapes, [1.0] * P)
    ref = OSH.pixelcnn_sample(ck["generator"], style, T, P, aud, noise, clip, shapes)
    assert torch.equal(codes[0::2], ref[0]) and torch.equal(codes[1::2], ref[0])
    assert torch.equal(kept[0::2], ref[2]) and torch.equal(kept[1::2], ref[2])
    assert (logp[0::2] - ref[1]).abs().max() <= 1e-6
    g3 = OG.pixelcnn_sample(ck["generator"], style2, T, P, aud2, noise, clip, shapes, [3.0] * P)[0]
    assert torch.equal(g3[0::2], g3[1::2]) and not torch.equal(g3[0::2], ref[0])


@pytest.fixture(scope="module")
def fix():
    return np.load(os.path.join(GOLDEN, "guided.npz"))


def fixture_inputs(z, case):
    """The inputs of fixture case ``case`` as the guided call takes them: B pairs, the clip's and the negative's features
    per pair, labels, the negative's label or speaker weights, per-pair settings and bias, the pair noise, the prefix."""
    s = z["settings"]
    B = len(s)
    neg = [str(n) for n in z["negative"]]
    styled = case == "style"
    spk = int(z["label_%s" % case])
    mfcc = torch.from_numpy(z["mfcc_%s" % case]).repeat(B, 1, 1)
    flat = torch.from_numpy(z["mfcc_neg_%s" % case]).repeat(B, 1, 1)
    na = [not styled and n in ("silence", "both") for n in neg]
    nl = [not styled and n in ("speaker", "both") for n in neg]
    gmfcc = torch.where(torch.tensor(na)[:, None, None], flat, mfcc)
    label = torch.full((B,), spk)
    glabel = torch.where(torch.tensor(nl), (label + 1) % 4, label)
    T = mfcc.shape[2] // 4
    out = dict(B=B, T=T, mfcc=mfcc, gmfcc=gmfcc, label=label, glabel=None if styled else glabel,
               gstyle=torch.full((B, 4), 0.25) if styled else None,
               kw=dict(temperature=s[:, 0].tolist(), top_k=[int(k) for k in s[:, 1]], top_p=s[:, 2].tolist(),
                       min_p=s[:, 3].tolist(), repetition_penalty=s[:, 4].tolist(),
                       repetition_window=[int(w) for w in s[:, 5]], code_bias=torch.from_numpy(z["bias_%s" % case])),
               guidance=s[:, 6].tolist(), noise=OSM.reference_noise(int(z["seed_%s" % case]), 2 * T, B), pre=None)
    if "pre_%s" % case in z:
        out["pre"] = torch.from_numpy(z["pre_%s" % case])
        mpre = torch.from_numpy(z["mfcc_pre_%s" % case]).repeat(B, 1, 1)
        out["mpre"], out["gmpre"] = mpre, torch.where(torch.tensor(na)[:, None, None], torch.zeros_like(mpre), mpre)
    return out


def test_fixture_is_the_checkpoints_and_is_unambiguous(fix):
    for case in ("3d", "style", "pre", "6d"):
        ck = synth.body_pixel_checkpoint_6d(0) if case == "6d" else synth.body_pixel_checkpoint(0)
        assert np.allclose(fix["fp_%s" % case], list(synth.fingerprint(ck).values()))
        assert (fix["kept_%s" % case] >= 1).all()
    assert float(fix["min_margin_top_p"]) >= 1e-5 and float(fix["min_margin_min_p"]) >= 1e-5
    w = fix["settings"][:, 6]
    assert set(w.tolist()) == {1.0, 0.5, 1.5, 2.0, 3.0} and set(fix["negative"].tolist()) == {"silence", "speaker", "both"}


@pytest.mark.parametrize("case", ["3d", "style", "pre", "6d"])
def test_oracle_reproduces_reference(fix, case):
    """the guided oracle, on 2P interleaved branches, draws the reference's codes and keep sizes bit for bit"""
    torch.set_grad_enabled(False)
    ck = synth.body_pixel_checkpoint_6d(0) if case == "6d" else synth.body_pixel_checkpoint(0)
    enc = lambda m: O.audio_encoder(ck["audioencoder"], m).unsqueeze(-1).repeat(1, 1, 1, 2)
    f = fixture_inputs(fix, case)
    B, T, kw = f["B"], f["T"], f["kw"]
    T0 = 0 if f["pre"] is None else f["pre"].shape[1]
    inter = lambda a, b: torch.stack([a, b], 1).reshape((2 * a.shape[0],) + tuple(a.shape[1:]))
    aud2 = enc(inter(f["mfcc"], f["gmfcc"]))
    if f["gstyle"] is not None:
        st = OST.onehot(f["label"], 4, T0 + T)
        style2 = inter(st, torch.full_like(st, 0.25))
    else:
        style2 = OST.onehot(inter(f["label"], f["glabel"]), 4, T0 + T)
    pre = {}
    if T0:
        pre = dict(pre_latents=f["pre"], pre_audio2=enc(inter(f["mpre"], f["gmpre"])))
    clip = list(zip(kw["temperature"], kw["top_k"], kw["top_p"], kw["min_p"]))
    shapes = list(zip(kw["repetition_penalty"], kw["repetition_window"]))
    codes, _, kept = OG.pixelcnn_sample(ck["generator"], style2, T, B, aud2, f["noise"], clip, shapes, f["guidance"],
                                        bias=kw["code_bias"], **pre)
    assert torch.equal(codes[0::2], codes[1::2])
    assert torch.equal(codes[0::2], torch.from_numpy(fix["codes_%s" % case])), case
    assert torch.equal(kept[0::2], torch.from_numpy(fix["kept_%s" % case])), case


def test_check_guidance():
    from talkshow_b200.engine import check_guidance

    assert check_guidance(2, 3).tolist() == [2.0] * 3 and check_guidance(2, 3).dtype == np.float32
    assert check_guidance([0, 1.5, 100], 3).tolist() == [0.0, 1.5, 100.0]
    assert check_guidance(torch.tensor([1.0, 2.0]), 2).tolist() == [1.0, 2.0]
    for bad, msg in ((-0.5, "clip 0"), (100.5, "clip 0"), (float("nan"), "clip 0"), (float("inf"), "clip 0"), (1e39, "clip 0"),
                     ([1.0, True], "clip 1"), ([1.0, "x"], "clip 1"), ([1.0, 2.0, 3.0], "3 per-clip"),
                     (np.ones((2, 1)), "one-dimensional")):
        with pytest.raises(ValueError, match=msg):
            check_guidance(bad, 2)


def test_unguided_calls_forward_as_before():
    e, rec = _engine()
    aud, label, mfcc = torch.zeros(2, 256, 5), torch.tensor([0, 1]), torch.zeros(2, 64, 20)
    noise = torch.ones(10, 2, 2048)
    # the same arguments as before: the caller's tensors, the sizes, no extra pointers (index 4 / 4 is the output buffer)
    ptr = lambda x: x.value if isinstance(x, C.c_void_p) else x
    e.pixelcnn_generate(aud, label, noise)
    name, a, _ = rec.calls[-1]
    assert name == "ts_pixelcnn_generate" and len(a) == 11
    assert [ptr(x) for x in a[1:4]] == [aud.data_ptr(), label.data_ptr(), noise.data_ptr()]
    assert [ptr(x) for x in a[5:]] == [None, 2, 5, None, 0, None]
    e.body_generate(mfcc, label, noise, guidance=None)
    name, a, _ = rec.calls[-1]
    assert name == "ts_body_generate" and len(a) == 9
    assert [ptr(x) for x in a[1:4]] == [mfcc.data_ptr(), label.data_ptr(), noise.data_ptr()] and list(a[6:8]) == [2, 20]
    e.pixelcnn_generate(aud, label, noise, temperature=0.7, want_logp=True, guidance=None)
    name, a, _ = rec.calls[-1]
    assert name == "ts_pixelcnn_sample" and len(a) == 14 and list(a[6:8]) == [2, 5]
    assert float(a[10]) == 0.7 and int(a[11]) == 0 and ptr(a[12]) is not None
    for kw, want in ((dict(), "generate"), (dict(temperature=0.7), "sample"), (dict(top_p=0.9), "sample_ctl"),
                     (dict(temperature=[0.7, 0.0]), "sample_clips"), (dict(repetition_penalty=2.0), "sample_shaped"),
                     (dict(guidance=None), "generate")):
        e.pixelcnn_generate(aud, label, noise, **kw)
        assert rec.calls[-1][0] == "ts_pixelcnn_" + want, kw
        e.body_generate(mfcc, label, noise, **kw)
        assert rec.calls[-1][0] == "ts_body_" + want, kw
    n = len(rec.calls)
    with pytest.raises(ValueError, match="need guidance"):
        e.pixelcnn_generate(aud, label, noise, guide_label=torch.tensor([1, 0]))
    with pytest.raises(ValueError, match="need guidance"):
        e.body_generate(mfcc, label, noise, guide_mfcc=mfcc)
    assert len(rec.calls) == n
    e.close()


def test_guided_calls_interleave_and_take_per_pair_inputs():
    e, rec = _engine()
    B = 3
    aud, label, mfcc = torch.zeros(B, 256, 5), torch.tensor([0, 1, 2]), torch.zeros(B, 64, 20)
    noise = torch.ones(10, B, 2048)
    for call, name in ((lambda **kw: e.pixelcnn_generate(aud, label, **kw), "ts_pixelcnn_sample_guided"),
                       (lambda **kw: e.body_generate(mfcc, label, **kw), "ts_body_sample_guided")):
        call(noise=noise, guidance=[1.0, 2.0, 0.5], guide_label=torch.tensor([3, 3, 3]), temperature=0.8, top_k=5)
        got, a, r = rec.calls[-1]
        assert got == name and r["P"] == B and r["guidance"].tolist() == [1.0, 2.0, 0.5]
        assert r["label"].tolist() == [0, 3, 1, 3, 2, 3] and not r["style"]
        assert r["ctl"] == (np.float32(0.8), 5, 1.0, 0.0) and r["clip"] is None and r["shape"] is None
        assert r["noise"] == noise.data_ptr()                 # one noise column per pair: the caller's tensor as it is
        call(noise=None, seeds=[5, 6, 7], guidance=2.0, guide_style=torch.full((B, 4), 0.25), repetition_penalty=[1.0, 2.0, 1.0],
             temperature=[0.5, 0.0, 1.0], code_bias=torch.zeros(2, 2048))
        got, a, r = rec.calls[-1]
        assert got == name and r["label"] is None and r["style"] and r["seeds"] and r["bias"]
        assert r["clip"]["temperature"].tolist() == [0.5, 0.0, 1.0] and r["shape"]["repetition_penalty"].tolist() == [1.0, 2.0, 1.0]
    n = len(rec.calls)
    for kw in (dict(guidance=2.0), dict(guidance=2.0, guide_label=label), dict(guidance=-1.0, guide_label=label + 1),
               dict(guidance=[1.0, 2.0], guide_label=label + 1)):
        with pytest.raises(ValueError):
            e.pixelcnn_generate(aud, label, noise=noise, **kw)
        with pytest.raises(ValueError):
            e.body_generate(mfcc, label, noise=noise, **kw)
    assert len(rec.calls) == n                                  # rejected before any call
    e.close()


def test_guided_style_from_labels():
    """a label clip against a schedule negative: both branches go in as schedules, the clip's as its one-hot rows"""
    e, rec = _engine()
    B, T = 2, 5
    e.pixelcnn_generate(torch.zeros(B, 256, T), torch.tensor([1, 2]), None, temperature=0.0, guidance=2.0,
                        guide_style=torch.full((B, 4), 0.25))
    got, a, r = rec.calls[-1]
    st = r["style_rows"]
    assert np.array_equal(st[0], np.eye(4, dtype=np.float32)[[1] * T]) and np.array_equal(st[2], np.eye(4, dtype=np.float32)[[2] * T])
    assert (st[1::2] == 0.25).all()
    e.close()


def test_chunks_hold_32_pairs():
    e, rec = _engine()
    B = 100
    w = np.linspace(0.0, 3.0, B)
    th = np.linspace(1.0, 2.0, B)
    e.pixelcnn_generate(torch.zeros(B, 256, 5), torch.arange(B) % 4, torch.ones(10, B, 2048), guidance=w,
                        guide_label=torch.full((B,), 3), repetition_penalty=th, want_logp=True, want_guide_logp=True)
    e.body_generate(torch.zeros(B, 64, 20), torch.arange(B) % 4, torch.ones(10, B, 2048), guidance=w,
                    guide_mfcc=torch.ones(B, 64, 20))
    names = [c[0] for c in rec.calls]
    assert names == ["ts_pixelcnn_sample_guided"] * 4 + ["ts_body_sample_guided"] * 4
    for i in (0, 4):
        calls = rec.calls[i:i + 4]
        assert [c[2]["P"] for c in calls] == [32, 32, 32, 4]
        assert np.array_equal(np.concatenate([c[2]["guidance"] for c in calls]), w.astype(np.float32))
        # per-branch conditioning advances by 64 rows, per-pair noise by 32 columns (a copy per chunk)
        assert calls[1][1][1] - calls[0][1][1] == 64 * (256 * 5 if i == 0 else 64 * 20) * 4
    assert np.array_equal(np.concatenate([c[2]["shape"]["repetition_penalty"] for c in rec.calls[:4]]), th.astype(np.float32))
    lab = np.concatenate([c[2]["label"] for c in rec.calls[:4]])
    assert lab[0::2].tolist() == (np.arange(B) % 4).tolist() and (lab[1::2] == 3).all()
    e.close()


class _KwEngine:
    """records the keywords of body_generate / pixelcnn_generate and answers with zeros"""

    def __init__(self):
        self.calls, self.pixelcnn_ncls = [], 4

    def latent_rows(self, M):
        return M // 4

    def vq_dim(self, which):
        return (39, 90)[which]

    def silence_mfcc(self, M, B=1):
        return torch.full((B, 64, M), -7.0)

    def audio_encode(self, mfcc):
        return torch.zeros(mfcc.shape[0], 256, mfcc.shape[2] // 4)

    def vq_decode(self, which, idx):
        return torch.zeros(idx.shape[0], (39, 90)[which], 4 * idx.shape[1])

    def body_generate(self, mfcc, label, noise, **kw):
        self.calls.append(("body_generate", mfcc, label, kw))
        B, T = mfcc.shape[0], mfcc.shape[2] // 4
        out = (torch.zeros(B, T, 2, dtype=torch.int64), torch.zeros(B, 4 * T, 129))
        return out + ((torch.zeros(B, T, 2),) if kw.get("want_logp") else ()) + (
            (torch.ones(B, T, 2),) if kw.get("want_guide_logp") else ())

    def pixelcnn_generate(self, aud, label, noise, **kw):
        self.calls.append(("pixelcnn_generate", aud, label, kw))
        B, T = aud.shape[0], kw.get("T") or aud.shape[2]
        out = (torch.zeros(B, T, 2, dtype=torch.int64),) + ((torch.zeros(B, T, 2),) if kw.get("want_logp") else ()) + (
            (torch.ones(B, T, 2),) if kw.get("want_guide_logp") else ())
        return out if len(out) > 1 else out[0]


def _wrapper(engine):
    import types

    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper

    g = TrainWrapper.__new__(TrainWrapper)
    g.engine, g.noise_device, g.noise_per_step = engine, "cpu", True
    g.args = types.SimpleNamespace(infer=True)
    return g


def test_wrappers_forward_the_guidance():
    e = _KwEngine()
    g = _wrapper(e)
    B, M = 2, 20
    mfcc, label = torch.zeros(B, 64, M), torch.tensor([0, 1])
    g.generate(mfcc, label, guidance=2.0, guide_mfcc="silence", temperature=0.0, keep_logp=True)
    _, _, _, kw = e.calls[-1]
    assert kw["guidance"] == 2.0 and kw["want_guide_logp"] and (kw["guide_mfcc"] == -7.0).all()
    assert kw["guide_mfcc"].shape == (B, 64, M) and (g.last_guide_logp == 1).all()
    g.generate(mfcc, label, guidance=[1.0, 3.0], guide_id=torch.tensor([2, 2]), temperature=0.0)
    _, _, _, kw = e.calls[-1]
    assert kw["guide_label"].tolist() == [2, 2] and not kw["want_guide_logp"] and g.last_guide_logp is None
    g.generate(mfcc, label, temperature=0.0)
    assert "guidance" not in e.calls[-1][3]                           # unguided: the keywords it forwarded before
    with pytest.raises(ValueError, match="needs guidance"):
        g.generate(mfcc, label, guide_id=torch.tensor([2, 2]), temperature=0.0)
    with pytest.raises(ValueError, match="silence"):
        g.generate(mfcc, label, guidance=2.0, guide_mfcc="noise", temperature=0.0)
    # infer: the negative audio goes through the audio encoder; "silence" from the front end
    g.infer(torch.zeros(B, M, 64), 0, label, B, temperature=0.0, guidance=2.0, guide_mfcc="silence")
    _, aud, _, kw = e.calls[-1]
    assert kw["guidance"] == 2.0 and kw["guide_aud"].shape == aud.shape and "guide_mfcc" not in kw
    g.infer(torch.zeros(B, M, 64), 0, label, B, temperature=0.0, guidance=2.0, guide_id=torch.tensor([3, 3]),
            pre_latents=torch.zeros(B, 2, 2, dtype=torch.int64), pre_audio=torch.ones(B, 256, 2, 2))
    _, aud, _, kw = e.calls[-1]
    assert kw["guide_aud"].shape == aud.shape and torch.equal(kw["guide_aud"], aud)   # the clip's own audio, prefix included
    with pytest.raises(ValueError, match="continuity"):
        g.infer_on_audio(np.zeros((M, 64), np.float32), continuity=True, guidance=2.0, guide_audio="silence")


def test_wholebody_and_sharded_forward_the_guidance(monkeypatch):
    from talkshow_b200.pipeline import WholeBody

    wb = WholeBody.__new__(WholeBody)
    seen = []
    monkeypatch.setattr(WholeBody, "generate", lambda self, mfcc, wave, label, **kw: seen.append((mfcc, label, kw)) or
                        torch.zeros(mfcc.shape[0], 3, 265))
    wb.e = _KwEngine()
    wb.device = "cpu"
    B, M = 5, 20
    mfcc = torch.arange(B, dtype=torch.float32)[:, None, None].expand(B, 64, M)
    gm = -mfcc
    w = [1.0, 1.5, 2.0, 2.5, 3.0]
    for rank, (lo, hi) in enumerate(((0, 3), (3, 5))):
        WholeBody.generate_sharded(wb, mfcc, torch.zeros(B, 16000), torch.arange(B), rank, 2, temperature=0.0,
                                   gather=False, guidance=w, guide_mfcc=gm, guide_label=3)
        m, lab, kw = seen[-1]
        assert kw["guidance"].tolist() == w[lo:hi] and torch.equal(kw["guide_mfcc"], gm[lo:hi])
        assert kw["guide_label"].tolist() == [3] * (hi - lo) and lab.tolist() == list(range(lo, hi))
    WholeBody.generate_sharded(wb, mfcc, torch.zeros(B, 16000), torch.arange(B), 0, 2, temperature=0.0, gather=False,
                               guidance=2.0, guide_mfcc="silence")
    assert seen[-1][2]["guide_mfcc"] == "silence"
    # a rank with no clips keeps no stale negative log p from an earlier call
    wb.last_guide_logp = torch.ones(1)
    WholeBody.generate_sharded(wb, mfcc[:1], torch.zeros(1, 16000), torch.arange(1), 1, 2, temperature=0.0, gather=False,
                               keep_logp=True, guidance=2.0, guide_label=3)
    assert tuple(wb.last_guide_logp.shape) == (0, M // 4, 2)
    with pytest.raises(ValueError):
        WholeBody.generate_sharded(wb, mfcc, torch.zeros(B, 16000), torch.arange(B), 0, 2, temperature=0.0, gather=False,
                                   guide_label=3)
