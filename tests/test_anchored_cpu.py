"""CPU (-m "not gpu"): anchored sampling of the body prior.

The rule of tests/oracle_anchored.py reproduces tests/golden/anchored.npz, made by the unmodified reference with pinned
draws (tests/golden/make_golden_anchored.py).  The host layer (validation, forwarding, wrappers, WholeBody, sharded
generation) runs on an oracle-backed stand-in engine that answers anchored calls with that rule."""
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
import oracle_anchored as OA  # noqa: E402
import oracle_sampling as OSM  # noqa: E402


def _fixture(geo):
    z = np.load(os.path.join(GOLDEN, "anchored.npz"))
    return {k[len(geo) + 1:]: z[k] for k in z.files if k.startswith(geo + "_")}


def _ckpts(geo):
    if geo == "6d":
        return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)
    return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0)


def _case(z, i):
    B, T = z["codes"].shape[1:3]
    t, k, p = (float(v) for v in z["setting"][i])
    return dict(temperature=t, top_k=int(k), top_p=p), torch.from_numpy(z["anchors"][i]), \
        OSM.reference_noise(int(z["seed"][i]), 2 * T, B)


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_oracle_reproduces_fixture(geo):
    torch.set_grad_enabled(False)
    z = _fixture(geo)
    ck, vq = _ckpts(geo)
    assert np.array_equal(z["fp"], np.array(list(synth.fingerprint(ck).values())))
    mfcc, label, stride = torch.from_numpy(z["mfcc"]), torch.from_numpy(z["label"]), int(z["pose_stride"])
    names = [str(n) for n in z["cases"]]
    assert len(names) == 21 and {n.split("/")[1] for n in names} == {"none", "prefix", "window", "body", "hand", "scattered", "all"}
    for i, name in enumerate(names):
        s, anchors, noise = _case(z, i)
        codes, poses, logp, kept, _ = OA.body_sample(ck, vq, mfcc, label, noise, anchors, s["temperature"], s["top_k"], s["top_p"])
        pin = OA.pinned(anchors)
        assert torch.equal(codes, torch.from_numpy(z["codes"][i])), name
        assert torch.equal(codes[pin], anchors[pin]) and (kept[pin] == 0).all(), name
        # the oracle's convolutions sum in another order than the reference's: its logits, and so log p, agree to ~1.5e-5
        assert (logp - torch.from_numpy(z["logp"][i])).abs().max() <= 5e-5, name
        assert (poses[:, ::stride] - torch.from_numpy(z["poses"][i])).abs().max() <= 1e-4, name
        if name.endswith("/all"):
            assert torch.equal(codes, anchors)
    # the patterns reuse the unanchored run's codes as anchors; the scattered one pins uniform random codes
    none = z["codes"][names.index(names[0])]
    for i, name in enumerate(names):
        a = z["anchors"][i]
        if name.endswith(("prefix", "window", "body", "hand", "all")):
            run0 = z["codes"][names.index(name.split("/")[0] + "/none")]
            assert (a[a >= 0] == run0[a >= 0]).all(), name
    assert none.shape == z["anchors"].shape[1:]


class AnchoredOracleEngine(OracleEngine):
    """OracleEngine whose sampling calls take the controls and ``anchors=`` of Engine and are answered by the rule of
    tests/oracle_anchored.py.  Every call is recorded in ``calls`` as (method, keyword names, anchors)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, temperature=1.0, top_k=0,
                          want_logp=False, top_p=1.0, min_p=0.0, want_kept=False, anchors=None):
        from talkshow_b200.engine import check_anchors

        kw = dict(temperature=temperature, top_k=top_k, want_logp=want_logp, top_p=top_p, want_kept=want_kept)
        B = aud.shape[0]
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        T = aud.shape[2] - T0 if T is None else T
        self.calls.append(("pixelcnn_generate", kw, None if anchors is None else check_anchors(anchors, B, T).clone()))
        a = torch.full((B, T, 2), -1, dtype=torch.int64) if anchors is None else check_anchors(anchors, B, T)
        a2 = aud.float().unsqueeze(-1).repeat(1, 1, 1, 2)
        label = label.reshape(-1).to(torch.int64).expand(B) if label.numel() == 1 else label.reshape(-1).to(torch.int64)
        pre = dict(pre_latents=pre_latents, pre_audio=a2[:, :, :T0]) if T0 else {}
        codes, logp, kept, _ = OA.pixelcnn_sample(self.sd["pixelcnn"], label, T, B, a2[:, :, T0:], noise, a, temperature, top_k,
                                                  top_p, min_p, window=self.window, **pre)
        out = (codes,) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())
        return out if len(out) > 1 else codes

    def body_generate(self, mfcc, label, noise, want_codes=True, temperature=1.0, top_k=0, want_logp=False, top_p=1.0,
                      min_p=0.0, want_kept=False, anchors=None):
        from talkshow_b200.engine import check_anchors

        B, T = mfcc.shape[0], self.latent_rows(mfcc.shape[2])
        self.calls.append(("body_generate", dict(want_codes=want_codes, temperature=temperature, top_k=top_k, top_p=top_p),
                           None if anchors is None else check_anchors(anchors, B, T).clone()))
        a = torch.full((B, T, 2), -1, dtype=torch.int64) if anchors is None else check_anchors(anchors, B, T)
        label = label.reshape(-1).to(torch.int64)
        label = label.expand(B) if label.numel() == 1 else label
        codes, poses, logp, kept, _ = OA.body_sample({"generator": self.sd["pixelcnn"], "audioencoder": self.sd["audioenc"]},
                                                     {"g_body": self.sd["vq0"], "g_hand": self.sd["vq1"]}, mfcc.float(), label,
                                                     noise, a, temperature, top_k, top_p, min_p, window=self.window)
        return ((codes if want_codes else None), poses) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())


def _wrapper(engine, geo="3d"):
    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Model.vq_path = ""
    cfg.Data.pose.convert_to_6d = geo == "6d"
    g = TrainWrapper(types.SimpleNamespace(gpu=0, infer=True), cfg, engine=engine)
    ck, vq = _ckpts(geo)
    g.load_state_dict(ck)
    g.load_vq_state_dict(vq)
    return g


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_wrappers_reproduce_fixture(geo):
    from talkshow_b200.pipeline import WholeBody

    torch.set_grad_enabled(False)
    z = _fixture(geo)
    e = AnchoredOracleEngine()
    g = _wrapper(e, geo)
    mfcc, label, stride = torch.from_numpy(z["mfcc"]), torch.from_numpy(z["label"]), int(z["pose_stride"])
    names = [str(n) for n in z["cases"]]
    for i in (names.index(n) for n in names if n.split("/")[1] in ("window", "scattered")):
        s, anchors, noise = _case(z, i)
        poses = g.generate(mfcc, label, noise_fn=lambda T, B: noise, anchors=anchors.numpy(), **s)
        assert torch.equal(g.last_codes, torch.from_numpy(z["codes"][i])), names[i]
        assert (poses[:, ::stride] - torch.from_numpy(z["poses"][i])).abs().max() <= 1e-4, names[i]
    # WholeBody keeps the codes it can be anchored to (the stand-in's face path is the 3-D net's)
    if geo == "3d":
        i = names.index([n for n in names if n.endswith("/hand")][0])
        s, anchors, noise = _case(z, i)
        ck, vq = _ckpts(geo)
        wb = WholeBody(e)
        wb.load(ck, vq, synth.face_checkpoint(0))
        B, M = mfcc.shape[0], mfcc.shape[2]
        wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(3))
        wb.generate(mfcc, wave, label, noise=noise, anchors=anchors, keep_codes=True, temperature=s["temperature"],
                    top_k=s["top_k"], top_p=s["top_p"])
        assert torch.equal(wb.last_codes, torch.from_numpy(z["codes"][i]))
    # pre_latents: the pinned rows before the free window as the prefix, the anchors of the rest over the chunk's rows
    i = names.index([n for n in names if n.endswith("/window")][0])
    s, anchors, noise = _case(z, i)
    T = anchors.shape[1]
    T0 = T // 3
    audio = e.audio_encode(mfcc)
    codes = e.pixelcnn_generate(audio, label, noise[2 * T0:], T=T - T0, pre_latents=anchors[:, :T0], anchors=anchors[:, T0:],
                                temperature=s["temperature"], top_k=s["top_k"], top_p=s["top_p"])
    assert torch.equal(codes, torch.from_numpy(z["codes"][i])[:, T0:])


def test_check_anchors():
    from talkshow_b200.engine import check_anchors

    t = torch.full((2, 3, 2), -1, dtype=torch.int64)
    assert check_anchors(t, 2, 3) is t
    t[0, 0, 0], t[1, 2, 1] = 0, 2047
    assert check_anchors(t, 2, 3) is t
    got = check_anchors(np.full((2, 3, 2), 7, dtype=np.int16), 2, 3)
    assert got.dtype == torch.int64 and (got == 7).all()
    assert check_anchors(np.zeros((2, 3, 2), dtype=np.uint64), 2, 3).dtype == torch.int64
    for bad in (torch.zeros(2, 3, 2, dtype=torch.int32), torch.zeros(2, 3, 2), torch.zeros(2, 3, dtype=torch.int64),
                torch.zeros(3, 3, 2, dtype=torch.int64), torch.zeros(2, 4, 2, dtype=torch.int64),
                torch.full((2, 3, 2), 2048, dtype=torch.int64), torch.full((2, 3, 2), -2, dtype=torch.int64),
                np.zeros((2, 3, 2), np.float64), np.full((2, 3, 2), 2 ** 63, dtype=np.uint64), [[[0, 0]] * 3] * 2, None, 5):
        with pytest.raises(ValueError):
            check_anchors(bad, 2, 3)


class _RecordingLib:
    """stands in for the C library: records which entry point a call reaches and returns success"""

    def __init__(self, real):
        self.real, self.names = real, []

    def __getattr__(self, name):
        if name.startswith(("ts_pixelcnn_", "ts_body_")) and name not in ("ts_pixelcnn_row_bytes",):
            return lambda *a: self.names.append(name) or 0
        return getattr(self.real, name)


def test_entry_points_and_validation():
    """anchors=None reaches the entry point the call reached before; anchors reach ts_*_sample_anchored; bad anchors raise
    ValueError before any call"""
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.L = rec = _RecordingLib(e.L)
    e._s = lambda: None
    e.latent_rows = lambda M: M // 4
    e.vq_dim = lambda which: (39, 90)[which]
    aud, label = torch.zeros(2, 256, 5), torch.tensor([0, 1])
    mfcc = torch.zeros(2, 64, 20)
    noise, seeds = torch.ones(10, 2, 2048), torch.tensor([1, 2])
    anchors = torch.full((2, 5, 2), -1, dtype=torch.int64)
    cases = [(dict(), "generate"), (dict(temperature=0.7), "sample"), (dict(top_p=0.9), "sample_ctl"),
             (dict(seeds=seeds), "sample_seeded"), (dict(anchors=anchors), "sample_anchored"),
             (dict(anchors=anchors, seeds=seeds, top_p=0.9, want_logp=True), "sample_anchored"),
             (dict(anchors=anchors.numpy(), temperature=0.0), "sample_anchored")]
    for kw, want in cases:
        n = None if "seeds" in kw or kw.get("temperature") == 0.0 else noise
        e.pixelcnn_generate(aud, label, n, **kw)
        assert rec.names[-1] == "ts_pixelcnn_" + want, kw
        e.body_generate(mfcc, label, n, **kw)
        assert rec.names[-1] == "ts_body_" + want, kw
    # a batch above the 64-sample tile: one call per chunk
    rec.names.clear()
    e.pixelcnn_generate(torch.zeros(65, 256, 5), torch.tensor([0]), torch.ones(10, 65, 2048),
                        anchors=torch.full((65, 5, 2), -1, dtype=torch.int64))
    assert rec.names == ["ts_pixelcnn_sample_anchored"] * 2
    rec.names.clear()
    for bad in (anchors.to(torch.int32), anchors[:, :4], torch.full((2, 5, 2), 2048, dtype=torch.int64), anchors.float()):
        with pytest.raises(ValueError):
            e.pixelcnn_generate(aud, label, noise, anchors=bad)
        with pytest.raises(ValueError):
            e.body_generate(mfcc, label, noise, anchors=bad)
    with pytest.raises(ValueError):
        e.pixelcnn_generate(aud, label, noise, seeds=seeds, anchors=anchors)      # two noise sources
    assert rec.names == []
    e.close()


def test_host_only_engine_refuses_anchored_entry_points():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.load_pixelcnn(synth.pixelcnn_state(0))
    L, h, n = e.L, e.h, None
    for name, args in (("ts_pixelcnn_sample_anchored", (h, n, n, n, n, n, n, n, 1, 2, n, 0, n, n)),
                       ("ts_body_sample_anchored", (h, n, n, n, n, n, n, n, 1, 8, n, n))):
        assert getattr(L, name)(*args) != 0 and b"host-only" in L.ts_last_error(h), name
    e.close()


def test_wrappers_forward_anchors_only_when_given(monkeypatch):
    from talkshow_b200.nets import smplx_body_pixel as bp

    torch.set_grad_enabled(False)
    e = AnchoredOracleEngine()
    g = _wrapper(e)
    B, M = 2, 16
    mfcc = synth.synth_mfcc(B, M, seed=4)
    label = torch.tensor([0, 1])
    g.noise_device = "cpu"
    g.generate(mfcc, label)
    assert e.calls[-1][2] is None
    anchors = torch.full((B, M // 4, 2), -1, dtype=torch.int64)
    anchors[1, 2, 0] = 17
    g.generate(mfcc, label, anchors=anchors)
    assert torch.equal(e.calls[-1][2], anchors) and g.last_codes[1, 2, 0] == 17
    feat = mfcc.transpose(1, 2)
    lat0, a0, _, _ = g.infer(feat, 0, label, B)
    assert e.calls[-1][2] is None
    lat1, _, _, _ = g.infer(feat, 0, label, B, lat0, a0, anchors=anchors)
    assert torch.equal(e.calls[-1][2], anchors) and lat1[1, 2, 0] == 17
    g.infer_on_audio(mfcc[0].transpose(0, 1).numpy(), B=2, anchors=anchors)
    assert torch.equal(e.calls[-1][2], anchors)
    monkeypatch.setattr(bp, "get_mfcc_sepa", lambda *a, **k: (np.zeros((32, 64), np.float32), 16))
    n = len(e.calls)
    with pytest.raises(ValueError):
        g.infer_on_audio("unused.wav", B=2, continuity=True, anchors=anchors)
    assert len(e.calls) == n
    with pytest.raises(ValueError):
        g.generate(mfcc, label, anchors=anchors[:, :3])


def test_wholebody_and_sharded_with_anchors():
    from talkshow_b200.pipeline import WholeBody, shard_range

    torch.set_grad_enabled(False)
    e = AnchoredOracleEngine()
    wb = WholeBody(e)
    wb.load(synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), synth.face_checkpoint(0))
    B, M = 5, 16
    mfcc = synth.synth_mfcc(B, M, seed=26)
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(27))
    label = torch.tensor([0, 1, 3, 2, 0])
    g = torch.Generator().manual_seed(28)
    anchors = torch.where(torch.rand(B, M // 4, 2, generator=g) < 0.5, torch.randint(0, 2048, (B, M // 4, 2), generator=g), -1)
    noise = OSM.reference_noise(29, 2 * (M // 4), B)
    one = wb.generate(mfcc, wave, label, noise=noise, anchors=anchors, keep_codes=True)
    codes = wb.last_codes
    assert e.calls[-1][1]["want_codes"] is True and torch.equal(codes[anchors >= 0], anchors[anchors >= 0])
    wb.generate(mfcc, wave, label, noise=noise)
    assert e.calls[-1][1]["want_codes"] is False and e.calls[-1][2] is None and wb.last_codes is None
    for world in (1, 2, 3):
        parts = []
        for r in range(world):
            parts.append(wb.generate_sharded(mfcc, wave, label, r, world, noise_full=noise, gather=False, anchors=anchors))
            lo, hi = shard_range(B, r, world)
            assert torch.equal(e.calls[-1][2], anchors[lo:hi]), (world, r)       # rank r passes its shard's anchors
        # the CPU stand-in's modules round differently at different batch sizes; the GPU test compares bit for bit
        assert (torch.cat(parts) - one).abs().max() <= 1e-5, world
    with pytest.raises(ValueError):
        wb.generate_sharded(mfcc, wave, label, 0, 2, noise_full=noise, anchors=anchors[:4])
