"""CPU (-m "not gpu"): sampling controls of the body prior (temperature, top-k, greedy, log-likelihood of each draw).

tests/golden/sampling.npz holds codes and poses of the unmodified reference's s2g_body_pixel.infer_on_audio with the
controlled warp in place of its softmax (tests/golden/make_golden_sampling.py).  The oracle (tests/oracle_sampling.py)
and the wrapper on an oracle-backed stand-in engine reproduce it; the host layer forwards the controls, validates them
and leaves the default calls on the default entry points."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle_engine import OracleEngine
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_sampling as OS  # noqa: E402


@pytest.fixture(scope="module")
def fix():
    return np.load(os.path.join(GOLDEN, "sampling.npz"))


def _ckpts(key):
    if key == "3d":
        return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0)
    return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)


def _case(fix, key, i):
    B = 3 if key == "3d" else 2
    mfcc = torch.from_numpy(fix["mfcc_%s" % key]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    t, k = fix["settings"][i].tolist()
    noise = None if t == 0 else OS.reference_noise(int(fix["seed"]) + i, 2 * T, B)
    return mfcc, torch.full((B,), int(fix["label_%s" % key])), noise, t, int(k)


def test_fixture_is_the_checkpoints(fix):
    for key in ("3d", "6d"):
        ck, vq = _ckpts(key)
        assert np.allclose(fix["fp_%s" % key], list(synth.fingerprint(ck).values()))
        assert np.allclose(fix["fp_vq_%s" % key], list(synth.fingerprint(vq).values()))


@pytest.mark.parametrize("key", ["3d", "6d"])
@pytest.mark.parametrize("i", range(5))
def test_oracle_reproduces_reference(fix, key, i):
    torch.set_grad_enabled(False)
    ck, vq = _ckpts(key)
    mfcc, label, noise, t, k = _case(fix, key, i)
    codes, poses, logp = OS.body_sample(ck, vq, mfcc, label, noise, t, k)
    assert torch.equal(codes, torch.from_numpy(fix["codes_%s_%d" % (key, i)]))
    assert (poses[:, ::int(fix["pose_stride"])] - torch.from_numpy(fix["poses_%s_%d" % (key, i)])).abs().max() <= 1e-5
    assert (logp <= 0).all() and torch.isfinite(logp).all()


class SamplingOracleEngine(OracleEngine):
    """OracleEngine plus the sampling controls of Engine.pixelcnn_generate / body_generate, answered by the oracle.
    Every call records its keyword arguments in ``calls``."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, **ctl):
        self.calls.append(("pixelcnn_generate", dict(ctl), noise is None))
        if not ctl:
            return super().pixelcnn_generate(aud, label, noise, T=T, pre_latents=pre_latents)
        B = aud.shape[0]
        a2 = aud.float().unsqueeze(-1).repeat(1, 1, 1, 2)
        label = label.reshape(-1).to(torch.int64).expand(B) if label.numel() == 1 else label.reshape(-1)
        t, k = ctl.get("temperature", 1.0), ctl.get("top_k", 0)
        if pre_latents is None:
            codes, logp = OS.pixelcnn_sample(self.sd["pixelcnn"], label, a2.shape[2], B, a2, noise, t, k, window=self.window)
        else:
            T0 = pre_latents.shape[1]
            codes, logp = OS.pixelcnn_sample(self.sd["pixelcnn"], label, a2.shape[2] - T0, B, a2[:, :, T0:], noise, t, k,
                                             pre_latents=pre_latents, pre_audio=a2[:, :, :T0], window=self.window)
        return (codes, logp) if ctl.get("want_logp") else codes

    def body_generate(self, mfcc, label, noise, want_codes=True, **ctl):
        self.calls.append(("body_generate", dict(ctl), noise is None))
        if not ctl:
            return super().body_generate(mfcc, label, noise, want_codes)
        B = mfcc.shape[0]
        label = label.reshape(-1).to(torch.int64)
        label = label.expand(B) if label.numel() == 1 else label
        codes, poses, logp = OS.body_sample({"generator": self.sd["pixelcnn"], "audioencoder": self.sd["audioenc"]},
                                            {"g_body": self.sd["vq0"], "g_hand": self.sd["vq1"]}, mfcc.float(), label,
                                            noise, ctl.get("temperature", 1.0), ctl.get("top_k", 0), window=self.window)
        out = (codes if want_codes else None, poses)
        return out + (logp,) if ctl.get("want_logp") else out


def _wrapper(key, engine):
    import types

    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Data.pose.convert_to_6d = key == "6d"
    cfg.Model.vq_path = ""
    ck, vq = _ckpts(key)
    g = TrainWrapper(types.SimpleNamespace(gpu=0, infer=True), cfg, engine=engine)
    g.load_state_dict(ck)
    g.load_vq_state_dict(vq)
    g.noise_device = "cpu"
    return g


@pytest.mark.parametrize("key,i", [("3d", 2), ("3d", 4), ("6d", 0), ("6d", 3), ("6d", 4)])
def test_wrapper_reproduces_reference(fix, key, i):
    torch.set_grad_enabled(False)
    e = SamplingOracleEngine()
    g = _wrapper(key, e)
    mfcc, label, noise, t, k = _case(fix, key, i)
    B = mfcc.shape[0]
    feat = mfcc[0].transpose(0, 1).numpy()                                     # (M, 64) features, as infer_on_audio takes them
    pred = g.infer_on_audio(feat, id=label[:1], B=B, temperature=t, top_k=k, keep_logp=True,
                            noise_fn=None if noise is None else (lambda T_, B_: noise))
    assert torch.equal(g.last_codes, torch.from_numpy(fix["codes_%s_%d" % (key, i)]))
    assert np.abs(pred[:, ::int(fix["pose_stride"])] - fix["poses_%s_%d" % (key, i)]).max() <= 1e-5
    assert g.last_logp.shape == g.last_codes.shape
    assert e.calls[-1] == ("body_generate", dict(temperature=t, top_k=k, want_logp=True), t == 0)


def test_defaults_use_default_entry_points():
    torch.set_grad_enabled(False)
    e = SamplingOracleEngine()
    g = _wrapper("6d", e)
    mfcc = synth.synth_mfcc(1, 16, seed=3)
    g.generate(mfcc, torch.tensor([1]), noise_fn=lambda T, B: torch.ones(2 * T, B, 2048))
    assert e.calls == [("body_generate", {}, False)] and g.last_logp is None
    lat, _, _, _ = g.infer(mfcc.transpose(1, 2), 0, torch.tensor([1]), 1)
    assert e.calls[-1] == ("pixelcnn_generate", {}, False)


def test_controls_forwarded_and_greedy_draws_no_noise():
    torch.set_grad_enabled(False)
    e = SamplingOracleEngine()
    g = _wrapper("6d", e)
    mfcc = synth.synth_mfcc(1, 16, seed=4)
    drawn = []
    g.generate(mfcc, torch.tensor([1]), noise_fn=lambda T, B: drawn.append(1), temperature=0.0)
    assert drawn == [] and e.calls[-1] == ("body_generate", dict(temperature=0.0, top_k=0, want_logp=False), True)
    noise = OS.reference_noise(5, 8, 1)
    g.generate(mfcc, torch.tensor([1]), noise_fn=lambda T, B: noise, temperature=0.9, top_k=7, keep_logp=True)
    assert e.calls[-1] == ("body_generate", dict(temperature=0.9, top_k=7, want_logp=True), False)
    assert g.last_logp.shape == (1, 4, 2)
    # the inner call of the continuity path: pre_latents / pre_audio conditioning with controls
    lat0, aud0, _, _ = g.infer(mfcc.transpose(1, 2), 0, torch.tensor([1]), 1, temperature=0.0, keep_logp=True)
    lp0 = g.last_logp
    lat1, _, _, _ = g.infer(mfcc.transpose(1, 2), 0, torch.tensor([1]), 1, lat0, aud0, temperature=0.0, keep_logp=True)
    assert e.calls[-1] == ("pixelcnn_generate", dict(temperature=0.0, top_k=0, want_logp=True), True)
    assert lp0.shape == lat0.shape and g.last_logp.shape == lat1.shape


def test_wholebody_forwards_controls():
    from talkshow_b200.pipeline import WholeBody

    torch.set_grad_enabled(False)
    e = SamplingOracleEngine()
    wb = WholeBody(e)
    ck, vq = _ckpts("3d")
    wb.load(ck, vq, synth.face_checkpoint(0))
    mfcc = synth.synth_mfcc(2, 16, seed=6)
    wave = torch.randn(2, 16000 * 16 // 30, generator=torch.Generator().manual_seed(7))
    label = torch.tensor([0, 1])
    out = wb.generate(mfcc, wave, label, temperature=0.0, top_k=3, keep_logp=True)
    assert e.calls[-1] == ("body_generate", dict(temperature=0.0, top_k=3, want_logp=True), True)
    assert out.shape[0] == 2 and wb.last_logp.shape == (2, 4, 2)
    noise = OS.reference_noise(8, 8, 2)
    wb.generate(mfcc, wave, label, noise=noise)
    assert e.calls[-1] == ("body_generate", {}, False) and wb.last_logp is None
    sh = wb.generate_sharded(mfcc, wave, label, 0, 1, noise_full=noise, temperature=1.2, top_k=9)
    assert e.calls[-1] == ("body_generate", dict(temperature=1.2, top_k=9, want_logp=False), False)
    assert torch.equal(sh, wb.generate(mfcc, wave, label, noise=noise, temperature=1.2, top_k=9))


@pytest.mark.parametrize("kw", [dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")),
                                dict(top_k=-1), dict(top_k=2049), dict(top_k=1.5), dict(temperature=0.5, noise=None)])
def test_invalid_controls_raise(kw):
    from talkshow_b200.engine import _controlled, check_sample_controls
    from talkshow_b200.pipeline import WholeBody

    kw = dict(kw)
    noise = kw.pop("noise", torch.ones(1))
    args = dict(temperature=1.0, top_k=0)
    args.update(kw)
    with pytest.raises(ValueError):
        _controlled(args["temperature"], args["top_k"], noise, False)
    if noise is not None:   # the wrappers draw their own noise: only the control values can be wrong there
        with pytest.raises(ValueError):
            check_sample_controls(args["temperature"], args["top_k"])
        e = SamplingOracleEngine()
        g = _wrapper("6d", e)
        with pytest.raises(ValueError):
            g.generate(synth.synth_mfcc(1, 16, seed=1), torch.tensor([0]), **args)
        with pytest.raises(ValueError):
            WholeBody(e).generate(synth.synth_mfcc(1, 16, seed=1), torch.zeros(1, 8533), torch.tensor([0]), **args)
        assert e.calls == []


@pytest.mark.parametrize("t", [1e-40, 1e-38, 1e-30])
def test_tiny_temperature_is_valid_and_draws_the_greedy_code(t):
    """Any finite temperature > 0 is accepted.  When logits / t overflows, the tempered softmax is NaN everywhere and the
    draw is the greedy code, never an index outside the codebook."""
    from talkshow_b200.engine import _controlled

    assert _controlled(t, 0, torch.ones(1), False) is True
    g = torch.Generator().manual_seed(9)
    logits = torch.randn(6, 2048, generator=g) * 8.0
    logits[1, 77] = logits[1].max() + 1.0                               # a clear maximum
    logits[2, :] = logits[2].max()                                      # every code tied: first index
    noise = torch.empty(6, 2048).exponential_(1, generator=g)
    greedy = OS.draw(logits, None, 0.0, 0)
    for k in (0, 5, 2048):
        code = OS.draw(logits, noise, t, k)
        assert ((code >= 0) & (code < 2048)).all()
        if t < 1e-38:                                                   # 1 / t alone overflows: every row falls back
            assert torch.equal(code, greedy)
        assert code[1] == 77 and code[2] in range(2048)


def test_sharded_world2_equals_one_engine():
    """rank 0 and rank 1 of a world-2 split, run without the gather on one stand-in engine, rebuild the single-engine
    result (to the stand-in's rounding): the full-batch noise is sliced per shard, and greedy decoding runs without noise on both shards."""
    from talkshow_b200.pipeline import WholeBody

    torch.set_grad_enabled(False)
    e = SamplingOracleEngine()
    wb = WholeBody(e)
    ck, vq = _ckpts("3d")
    wb.load(ck, vq, synth.face_checkpoint(0))
    B = 3
    mfcc = synth.synth_mfcc(B, 16, seed=16)
    wave = torch.randn(B, 16000 * 16 // 30, generator=torch.Generator().manual_seed(17))
    label = torch.tensor([0, 1, 3])
    noise = OS.reference_noise(18, 8, B)
    for t, k in [(0.8, 7), (0.0, 0)]:
        nz = None if t == 0 else noise
        one = wb.generate(mfcc, wave, label, noise=nz, temperature=t, top_k=k, keep_logp=True)
        lp1 = wb.last_logp
        parts, lps = [], []
        for r in range(2):
            parts.append(wb.generate_sharded(mfcc, wave, label, r, 2, noise_full=nz, gather=False, temperature=t, top_k=k,
                                             keep_logp=True))
            lps.append(wb.last_logp)
        # the CPU stand-in's modules round differently at different batch sizes; the GPU test compares bit for bit
        assert (torch.cat(parts) - one).abs().max() <= 1e-5 and (torch.cat(lps) - lp1).abs().max() <= 1e-5
