"""CPU (-m "not gpu"): styled sampling of the body prior (per-row mixtures of the speaker embeddings).

The rule of tests/oracle_style.py reproduces tests/golden/style.npz, made by the unmodified reference with each layer's
class embedding swapped for the blend (tests/golden/make_golden_style.py).  The host layer (validation, forwarding,
wrappers, WholeBody, sharded generation) runs on an oracle-backed stand-in engine that answers styled calls with that
rule."""
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
import oracle_sampling as OSM  # noqa: E402
import oracle_style as OST  # noqa: E402
import talkshow_oracle as O  # noqa: E402


def _fixture(geo):
    z = np.load(os.path.join(GOLDEN, "style.npz"))
    return {k[len(geo) + 1:]: z[k] for k in z.files if k.startswith(geo + "_")}


def _ckpts(geo):
    if geo == "6d":
        return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)
    return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0)


@pytest.mark.parametrize("geo", ["3d", "6d"])
def test_oracle_reproduces_fixture(geo):
    torch.set_grad_enabled(False)
    z = _fixture(geo)
    ck, _ = _ckpts(geo)
    assert np.array_equal(z["fp"], np.array(list(synth.fingerprint(ck).values())))
    names = [str(n) for n in z["cases"]]
    assert names == ["onehot0", "onehot1", "onehot2", "onehot3", "half02", "three1_13", "uniform", "nine1_20", "mixed"]
    audio = torch.from_numpy(z["audio"]).unsqueeze(-1).repeat(1, 1, 1, 2)
    B, T = z["codes"].shape[1:3]
    for i, name in enumerate(names):
        w = torch.from_numpy(z["weights"][i])
        noise = OSM.reference_noise(int(z["seed"][i]), 2 * T, B)
        codes, logp, _ = OST.pixelcnn_sample(ck["generator"], w[:, None].expand(B, T, 4), T, B, audio, noise)
        assert torch.equal(codes, torch.from_numpy(z["codes"][i])), name
        # the oracle's convolutions sum in another order than the reference's (as in test_anchored_cpu)
        assert (logp - torch.from_numpy(z["logp"][i])).abs().max() <= 5e-5, name
    # the blends are convex, and the one-hot cases are plain labels
    assert np.allclose(z["weights"].sum(-1), 1) and (z["weights"] >= 0).all()


def test_oracle_onehot_equals_label_and_is_causal():
    torch.set_grad_enabled(False)
    sd = synth.pixelcnn_state(0)
    B, T = 3, 8
    g = torch.Generator().manual_seed(11)
    x = torch.randint(0, 2048, (B, T, 2), generator=g)
    aud = torch.randn(B, 256, T, 2, generator=g)
    for s in range(4):
        label = torch.full((B,), s, dtype=torch.int64)
        assert torch.equal(OST.pixelcnn_forward(sd, x, OST.onehot(label, 4, T), aud), O.pixelcnn_forward(sd, x, label, aud))
    # a schedule that switches at row k: the draws before k equal the constant schedule's
    k = 4
    a = torch.tensor([0.5, 0.0, 0.5, 0.0])
    b = torch.tensor([0.0, 0.75, 0.0, 0.25])
    const = a.expand(B, T, 4).clone()
    switch = const.clone()
    switch[:, k:] = b
    noise = OSM.reference_noise(12, 2 * T, B)
    c0, l0, _ = OST.pixelcnn_sample(sd, const, T, B, aud, noise)
    c1, l1, _ = OST.pixelcnn_sample(sd, switch, T, B, aud, noise)
    assert torch.equal(c0[:, :k], c1[:, :k]) and torch.equal(l0[:, :k], l1[:, :k])
    assert not torch.equal(l0[:, k:], l1[:, k:])


def test_check_style():
    from talkshow_b200.engine import check_style

    w = torch.tensor([[0.25, 0.25, 0.5, 0.0], [1.0, 0.0, 0.0, 0.0]])
    got = check_style(w, 2, 3, 4)
    assert got.shape == (2, 3, 4) and got.dtype == torch.float32 and torch.equal(got[:, 1], w)
    full = torch.rand(2, 3, 4, dtype=torch.float64)
    full /= full.sum(-1, keepdim=True)
    got = check_style(full.numpy(), 2, 3, 4)
    assert got.dtype == torch.float32 and torch.equal(got, full.float())
    assert check_style(np.tile(np.float16([0.5, 0.5, 0, 0]), (2, 1)), 2, 3, 4).dtype == torch.float32
    off = torch.full((2, 3, 4), 0.25)
    off[1, 2, 0] += 2e-5
    nan, neg = torch.full((2, 3, 4), 0.25), torch.full((2, 3, 4), 0.25)
    nan[0, 0, 0] = float("nan")
    neg[0, 1, :2] = torch.tensor([-0.25, 0.75])
    for bad in (torch.full((2, 3, 4), 0.25, dtype=torch.float64)[:, :2], torch.full((2, 3, 5), 0.2),
                torch.full((3, 3, 4), 0.25), torch.full((2, 4), 0.25)[:1], torch.ones(2, 3, 4, dtype=torch.int64),
                np.ones((2, 4), np.int32), off, nan, neg, torch.full((2, 3, 4), float("inf")), [[0.25] * 4] * 2, None, 1.0):
        with pytest.raises(ValueError):
            check_style(bad, 2, 3, 4)
    with pytest.raises(ValueError):                 # the prior's class count decides ncls
        check_style(torch.full((2, 3, 4), 0.25), 2, 3, 5)


class _RecordingLib:
    """stands in for the C library: records which entry point a call reaches, with its arguments, and returns success"""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        if name.startswith(("ts_pixelcnn_", "ts_body_")) and name not in ("ts_pixelcnn_row_bytes",):
            return lambda *a: self.calls.append((name, a)) or 0
        return getattr(self.real, name)


def test_entry_points_and_validation():
    """style=None reaches the entry point the call reached before with the same arguments; style reaches the styled entry
    points, chunked with the batch; bad styles raise ValueError before any call"""
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.load_pixelcnn(synth.pixelcnn_state(0))
    assert e.pixelcnn_ncls == 4
    e.L = rec = _RecordingLib(e.L)
    e._s = lambda: None
    e.latent_rows = lambda M: M // 4
    e.vq_dim = lambda which: (39, 90)[which]
    aud, label, mfcc = torch.zeros(2, 256, 5), torch.tensor([0, 1]), torch.zeros(2, 64, 20)
    noise, seeds = torch.ones(10, 2, 2048), torch.tensor([1, 2])
    anchors = torch.full((2, 5, 2), -1, dtype=torch.int64)
    style = torch.full((2, 5, 4), 0.25)
    for kw, want in [(dict(), "generate"), (dict(temperature=0.7), "sample"), (dict(top_p=0.9), "sample_ctl"),
                     (dict(seeds=seeds), "sample_seeded"), (dict(anchors=anchors), "sample_anchored")]:
        n = None if "seeds" in kw else noise
        e.pixelcnn_generate(aud, label, n, **kw)
        assert rec.calls[-1][0] == "ts_pixelcnn_" + want, kw
        e.body_generate(mfcc, label, n, **kw)
        assert rec.calls[-1][0] == "ts_body_" + want, kw
    e.pixelcnn_score(aud, label, torch.zeros(2, 5, 2, dtype=torch.int64))
    assert rec.calls[-1][0] == "ts_pixelcnn_score"
    for kw in (dict(style=style), dict(style=style[:, 0].numpy(), seeds=seeds, top_p=0.9, want_logp=True),
               dict(style=style, anchors=anchors, temperature=0.0)):
        n = None if "seeds" in kw or kw.get("temperature") == 0.0 else noise
        e.pixelcnn_generate(aud, None, n, **kw)
        name, a = rec.calls[-1]
        assert name == "ts_pixelcnn_sample_styled" and a[2].value is None and a[4] == 4, kw
        e.body_generate(mfcc, label, n, **kw)
        assert rec.calls[-1][0] == "ts_body_sample_styled" and rec.calls[-1][1][4] == 4, kw
    e.pixelcnn_score(aud, None, torch.zeros(2, 5, 2, dtype=torch.int64), style=style)
    assert rec.calls[-1][0] == "ts_pixelcnn_score_styled" and rec.calls[-1][1][4] == 4
    # with pre_latents the schedule covers the prefix too
    e.pixelcnn_generate(torch.zeros(2, 256, 7), label, noise, T=5, pre_latents=torch.zeros(2, 2, 2, dtype=torch.int64),
                        style=torch.full((2, 7, 4), 0.25))
    assert rec.calls[-1][0] == "ts_pixelcnn_sample_styled"
    # a batch above the 64-sample tile: one call per chunk, each with its clips' rows
    rec.calls.clear()
    big = torch.zeros(65, 5, 4)
    big[:, :, 1] = 1
    big[64, :, 1], big[64, :, 3] = 0, 1
    e.pixelcnn_generate(torch.zeros(65, 256, 5), torch.tensor([0]), torch.ones(10, 65, 2048), style=big)
    assert [c[0] for c in rec.calls] == ["ts_pixelcnn_sample_styled"] * 2
    assert [c[1][10] for c in rec.calls] == [64, 1]
    rec.calls.clear()
    for bad in (style[:, :4], torch.full((2, 5, 3), 1 / 3), style * 2, -style, style.to(torch.int64)):
        for call in (lambda: e.pixelcnn_generate(aud, label, noise, style=bad), lambda: e.body_generate(mfcc, label, noise, style=bad),
                     lambda: e.pixelcnn_score(aud, label, torch.zeros(2, 5, 2, dtype=torch.int64), style=bad)):
            with pytest.raises(ValueError):
                call()
    with pytest.raises(ValueError):
        e.pixelcnn_generate(aud, None, noise)       # a label or a style
    assert rec.calls == []
    e.close()


def test_host_only_engine_refuses_styled_entry_points():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.load_pixelcnn(synth.pixelcnn_state(0))
    L, h, n = e.L, e.h, None
    for name, args in (("ts_pixelcnn_sample_styled", (h, n, n, n, 4, n, n, n, n, n, 1, 2, n, 0, n, n)),
                       ("ts_body_sample_styled", (h, n, n, n, 4, n, n, n, n, n, 1, 8, n, n)),
                       ("ts_pixelcnn_score_styled", (h, n, n, n, 4, n, n, n, 1, 2, n))):
        assert getattr(L, name)(*args) != 0 and b"host-only" in L.ts_last_error(h), name
    e.close()


class StyledOracleEngine(OracleEngine):
    """OracleEngine whose sampling calls take the controls, ``anchors=`` and ``style=`` of Engine and are answered by the
    rule of tests/oracle_style.py (a labelled call by its one-hot schedule).  Every call is recorded in ``calls`` as
    (method, keyword names, style or None)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    def load_pixelcnn(self, sd):
        super().load_pixelcnn(sd)
        self.pixelcnn_ncls = sd["layers.0.class_cond_embedding.weight"].shape[0]

    def _style(self, style, label, B, H):
        from talkshow_b200.engine import check_style

        if style is not None:
            return check_style(style, B, H, self.pixelcnn_ncls)
        label = label.reshape(-1).to(torch.int64)
        return OST.onehot(label.expand(B) if label.numel() == 1 else label, self.pixelcnn_ncls, H)

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, temperature=1.0, top_k=0,
                          want_logp=False, top_p=1.0, min_p=0.0, want_kept=False, anchors=None, style=None):
        B = aud.shape[0]
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        T = aud.shape[2] - T0 if T is None else T
        st = self._style(style, label, B, T0 + T)
        self.calls.append(("pixelcnn_generate", dict(temperature=temperature), None if style is None else st.clone()))
        a2 = aud.float().unsqueeze(-1).repeat(1, 1, 1, 2)
        pre = dict(pre_latents=pre_latents, pre_audio=a2[:, :, :T0]) if T0 else {}
        codes, logp, kept = OST.pixelcnn_sample(self.sd["pixelcnn"], st, T, B, a2[:, :, T0:], noise, temperature, top_k, top_p,
                                                min_p, anchors=anchors, window=self.window, **pre)
        out = (codes,) + ((logp,) if want_logp else ()) + ((kept,) if want_kept else ())
        return out if len(out) > 1 else codes

    def body_generate(self, mfcc, label, noise, want_codes=True, temperature=1.0, top_k=0, want_logp=False, top_p=1.0,
                      min_p=0.0, want_kept=False, anchors=None, style=None):
        B, T = mfcc.shape[0], self.latent_rows(mfcc.shape[2])
        st = self._style(style, label, B, T)
        self.calls.append(("body_generate", dict(want_codes=want_codes), None if style is None else st.clone()))
        codes, poses, logp, kept = OST.body_sample({"generator": self.sd["pixelcnn"], "audioencoder": self.sd["audioenc"]},
                                                   {"g_body": self.sd["vq0"], "g_hand": self.sd["vq1"]}, mfcc.float(), st,
                                                   noise, temperature, top_k, top_p, min_p, anchors=anchors,
                                                   window=self.window)
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


def test_wrapper_reproduces_fixture():
    torch.set_grad_enabled(False)
    z = _fixture("3d")
    e = StyledOracleEngine()
    g = _wrapper(e)
    names = [str(n) for n in z["cases"]]
    mfcc = torch.from_numpy(z["mfcc"])
    B, T = z["codes"].shape[1:3]
    for name in ("onehot2", "mixed"):
        i = names.index(name)
        noise = OSM.reference_noise(int(z["seed"][i]), 2 * T, B)
        g.generate(mfcc, torch.tensor([0]), noise_fn=lambda T_, B_: noise, style=torch.from_numpy(z["weights"][i]))
        assert torch.equal(g.last_codes, torch.from_numpy(z["codes"][i])), name


def test_wrappers_forward_style_only_when_given(monkeypatch):
    from talkshow_b200.nets import smplx_body_pixel as bp

    torch.set_grad_enabled(False)
    e = StyledOracleEngine()
    g = _wrapper(e)
    g.noise_device = "cpu"
    B, M = 2, 16
    T = M // 4
    mfcc = synth.synth_mfcc(B, M, seed=4)
    label = torch.tensor([0, 1])
    style = torch.zeros(B, T, 4)
    style[:, :2, 0] = 1
    style[:, 2:, 3] = 1
    g.generate(mfcc, label)
    assert e.calls[-1][2] is None
    g.generate(mfcc, label, style=style)
    assert torch.equal(e.calls[-1][2], style)
    feat = mfcc.transpose(1, 2)
    lat0, a0, _, _ = g.infer(feat, 0, label, B)
    assert e.calls[-1][2] is None
    style2 = torch.cat([style, style], 1)
    g.infer(feat, 0, label, B, lat0, a0, style=style2)
    assert torch.equal(e.calls[-1][2], style2)              # prefix rows and chunk rows
    g.infer_on_audio(mfcc[0].transpose(0, 1).numpy(), B=2, style=style)
    assert torch.equal(e.calls[-1][2], style)
    # continuity: chunk 0 gets rows [0, T_a), chunk 1 all T_a + T_b rows
    monkeypatch.setattr(bp, "get_mfcc_sepa", lambda *a, **k: (np.asarray(synth.synth_mfcc(1, 40, seed=5)[0].T), 16))
    full = torch.rand(B, 10, 4, generator=torch.Generator().manual_seed(6))
    full /= full.sum(-1, keepdim=True)
    n = len(e.calls)
    g.infer_on_audio("unused.wav", B=2, continuity=True, style=full)
    assert len(e.calls) == n + 2
    assert torch.equal(e.calls[-2][2], full[:, :4]) and torch.equal(e.calls[-1][2], full)
    with pytest.raises(ValueError):
        g.infer_on_audio("unused.wav", B=2, continuity=True, style=full[:, :9])
    with pytest.raises(ValueError):
        g.generate(mfcc, label, style=style[:, :3])


def test_wholebody_and_sharded_with_style():
    from talkshow_b200.pipeline import WholeBody, shard_range

    torch.set_grad_enabled(False)
    e = StyledOracleEngine()
    wb = WholeBody(e)
    wb.load(synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), synth.face_checkpoint(0))
    B, M = 5, 16
    T = M // 4
    mfcc = synth.synth_mfcc(B, M, seed=26)
    wave = torch.randn(B, 16000 * M // 30, generator=torch.Generator().manual_seed(27))
    label = torch.tensor([0, 1, 3, 2, 0])
    style = torch.rand(B, T, 4, generator=torch.Generator().manual_seed(28))
    style /= style.sum(-1, keepdim=True)
    noise = OSM.reference_noise(29, 2 * T, B)
    one = wb.generate(mfcc, wave, label, noise=noise, style=style)
    assert torch.equal(e.calls[-1][2], style)
    labelled = wb.generate(mfcc, wave, label, noise=noise)
    assert e.calls[-1][2] is None
    onehot = wb.generate(mfcc, wave, label, noise=noise, style=OST.onehot(label, 4, T))
    assert torch.equal(onehot, labelled)
    for world in (1, 2, 3):
        parts = []
        for r in range(world):
            parts.append(wb.generate_sharded(mfcc, wave, label, r, world, noise_full=noise, gather=False, style=style))
            lo, hi = shard_range(B, r, world)
            assert torch.equal(e.calls[-1][2], style[lo:hi]), (world, r)          # rank r passes its shard's rows
        # the CPU stand-in's modules round differently at different batch sizes; the GPU test compares bit for bit
        assert (torch.cat(parts) - one).abs().max() <= 1e-5, world
    with pytest.raises(ValueError):
        wb.generate_sharded(mfcc, wave, label, 0, 2, noise_full=noise, style=style[:4])
