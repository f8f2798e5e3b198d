"""CPU (-m "not gpu"): nucleus (top-p) and min-p sampling of the body prior.

tests/golden/sampling_p.npz holds codes, keep-set sizes and poses of the unmodified reference's
s2g_body_pixel.infer_on_audio with the warp in place of its softmax (tests/golden/make_golden_nucleus.py).  The oracle
(tests/oracle_nucleus.py) and the wrappers on an oracle-backed stand-in engine reproduce it; the integer keep rule agrees
with the float64 sort-and-cumsum rule away from the threshold; the host layer forwards the controls, validates them and
leaves every call without them on the entry points it used before."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle_engine import OracleEngine
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_nucleus as ON  # noqa: E402
import oracle_sampling as OS  # noqa: E402

NSET = 6


@pytest.fixture(scope="module")
def fix():
    return np.load(os.path.join(GOLDEN, "sampling_p.npz"))


def _ckpts(key):
    if key == "3d":
        return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0)
    return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0)


def _case(fix, key, i):
    B = 3 if key == "3d" else 2
    mfcc = torch.from_numpy(fix["mfcc_%s" % key]).repeat(B, 1, 1)
    T = mfcc.shape[2] // 4
    t, k, p, m = fix["settings"][i].tolist()
    noise = OS.reference_noise(int(fix["seeds_%s" % key][i]), 2 * T, B)
    return mfcc, torch.full((B,), int(fix["label_%s" % key])), noise, dict(temperature=t, top_k=int(k), top_p=p, min_p=m)


def test_fixture_is_the_checkpoints_and_is_unambiguous(fix):
    for key in ("3d", "6d"):
        ck, vq = _ckpts(key)
        assert np.allclose(fix["fp_%s" % key], list(synth.fingerprint(ck).values()))
        assert np.allclose(fix["fp_vq_%s" % key], list(synth.fingerprint(vq).values()))
    assert len(fix["settings"]) == NSET
    assert float(fix["min_margin_top_p"]) >= 1e-5 and float(fix["min_margin_min_p"]) >= 1e-5


@pytest.mark.parametrize("key", ["3d", "6d"])
@pytest.mark.parametrize("i", range(NSET))
def test_oracle_reproduces_reference(fix, key, i):
    torch.set_grad_enabled(False)
    ck, vq = _ckpts(key)
    mfcc, label, noise, ctl = _case(fix, key, i)
    codes, poses, logp, kept, margin = ON.body_sample(ck, vq, mfcc, label, noise, **ctl)
    assert torch.equal(codes, torch.from_numpy(fix["codes_%s_%d" % (key, i)]))
    assert torch.equal(kept, torch.from_numpy(fix["kept_%s_%d" % (key, i)]))
    assert (poses[:, ::int(fix["pose_stride"])] - torch.from_numpy(fix["poses_%s_%d" % (key, i)])).abs().max() <= 1e-5
    assert (logp <= 0).all() and torch.isfinite(logp).all()
    if i == NSET - 1:                                       # top_p -> 0 decodes greedily
        greedy, _, _, gk, _ = ON.body_sample(ck, vq, mfcc, label, None, temperature=0.0)
        assert torch.equal(codes, greedy) and (kept == 1).all() and (gk == 1).all()


class NucleusOracleEngine(OracleEngine):
    """OracleEngine plus the sampling controls of Engine.pixelcnn_generate / body_generate (top_p, min_p and want_kept
    included), answered by the oracle.  Every call records its keyword arguments in ``calls``."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    @staticmethod
    def _args(ctl):
        return [ctl.get("temperature", 1.0), ctl.get("top_k", 0), ctl.get("top_p", 1.0), ctl.get("min_p", 0.0)]

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, **ctl):
        self.calls.append(("pixelcnn_generate", dict(ctl), noise is None))
        if not ctl:
            return super().pixelcnn_generate(aud, label, noise, T=T, pre_latents=pre_latents)
        B = aud.shape[0]
        a2 = aud.float().unsqueeze(-1).repeat(1, 1, 1, 2)
        label = label.reshape(-1).to(torch.int64).expand(B) if label.numel() == 1 else label.reshape(-1)
        if pre_latents is None:
            codes, logp, kept, _ = ON.pixelcnn_sample(self.sd["pixelcnn"], label, a2.shape[2], B, a2, noise, *self._args(ctl),
                                                      window=self.window)
        else:
            T0 = pre_latents.shape[1]
            codes, logp, kept, _ = ON.pixelcnn_sample(self.sd["pixelcnn"], label, a2.shape[2] - T0, B, a2[:, :, T0:], noise,
                                                      *self._args(ctl), pre_latents=pre_latents, pre_audio=a2[:, :, :T0],
                                                      window=self.window)
        out = (codes,) + ((logp,) if ctl.get("want_logp") else ()) + ((kept,) if ctl.get("want_kept") else ())
        return out if len(out) > 1 else codes

    def body_generate(self, mfcc, label, noise, want_codes=True, **ctl):
        self.calls.append(("body_generate", dict(ctl), noise is None))
        if not ctl:
            return super().body_generate(mfcc, label, noise, want_codes)
        B = mfcc.shape[0]
        label = label.reshape(-1).to(torch.int64)
        label = label.expand(B) if label.numel() == 1 else label
        codes, poses, logp, kept, _ = ON.body_sample({"generator": self.sd["pixelcnn"], "audioencoder": self.sd["audioenc"]},
                                                     {"g_body": self.sd["vq0"], "g_hand": self.sd["vq1"]}, mfcc.float(), label,
                                                     noise, *self._args(ctl), window=self.window)
        return ((codes if want_codes else None, poses) + ((logp,) if ctl.get("want_logp") else ())
                + ((kept,) if ctl.get("want_kept") else ()))


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


@pytest.mark.parametrize("key,i", [("3d", 0), ("6d", 2), ("6d", 3), ("6d", 4)])
def test_wrapper_reproduces_reference(fix, key, i):
    torch.set_grad_enabled(False)
    e = NucleusOracleEngine()
    g = _wrapper(key, e)
    mfcc, label, noise, ctl = _case(fix, key, i)
    feat = mfcc[0].transpose(0, 1).numpy()
    pred = g.infer_on_audio(feat, id=label[:1], B=mfcc.shape[0], keep_logp=True, noise_fn=lambda T_, B_: noise, **ctl)
    assert torch.equal(g.last_codes, torch.from_numpy(fix["codes_%s_%d" % (key, i)]))
    assert torch.equal(g.last_kept, torch.from_numpy(fix["kept_%s_%d" % (key, i)]))
    assert np.abs(pred[:, ::int(fix["pose_stride"])] - fix["poses_%s_%d" % (key, i)]).max() <= 1e-5
    assert g.last_logp.shape == g.last_codes.shape
    assert e.calls[-1] == ("body_generate", dict(ctl, want_logp=True, want_kept=True), False)


def test_controls_forwarded_and_defaults_unchanged():
    from talkshow_b200.engine import _controlled, _needs_ctl, sample_controls

    torch.set_grad_enabled(False)
    assert sample_controls() == {} and sample_controls(1.0, 0, False, 1.0, 0.0) == {}
    assert sample_controls(0.7, 5, True) == dict(temperature=0.7, top_k=5, want_logp=True)      # no new key without top_p / min_p
    assert sample_controls(top_p=0.9) == dict(temperature=1.0, top_k=0, want_logp=False, top_p=0.9, min_p=0.0, want_kept=False)
    assert sample_controls(min_p=0.1, keep_logp=True)["want_kept"] is True
    assert _controlled(1.0, 0, torch.ones(1), False) is False and not _needs_ctl(1.0, 0.0, False)
    assert _controlled(1.0, 0, torch.ones(1), False, 0.9, 0.0) is True and _needs_ctl(0.9, 0.0, False)
    assert _controlled(1.0, 0, torch.ones(1), False, want_kept=True) is True and _needs_ctl(1.0, 0.0, True)
    e = NucleusOracleEngine()
    g = _wrapper("6d", e)
    mfcc = synth.synth_mfcc(1, 16, seed=3)
    noise = OS.reference_noise(5, 8, 1)
    g.generate(mfcc, torch.tensor([1]), noise_fn=lambda T, B: noise)
    assert e.calls == [("body_generate", {}, False)] and g.last_logp is None and g.last_kept is None
    g.generate(mfcc, torch.tensor([1]), noise_fn=lambda T, B: noise, temperature=0.9, keep_logp=True)
    assert e.calls[-1] == ("body_generate", dict(temperature=0.9, top_k=0, want_logp=True), False) and g.last_kept is None
    g.generate(mfcc, torch.tensor([1]), noise_fn=lambda T, B: noise, top_p=0.8)
    assert e.calls[-1][1] == dict(temperature=1.0, top_k=0, want_logp=False, top_p=0.8, min_p=0.0, want_kept=False)
    assert g.last_kept is None and g.last_logp is None
    # the inner call of the continuity path, with pre_latents / pre_audio conditioning
    lat0, aud0, _, _ = g.infer(mfcc.transpose(1, 2), 0, torch.tensor([1]), 1, noise_fn=lambda T, B: noise, min_p=0.2, keep_logp=True)
    k0 = g.last_kept
    lat1, _, _, _ = g.infer(mfcc.transpose(1, 2), 0, torch.tensor([1]), 1, lat0, aud0, noise_fn=lambda T, B: noise, min_p=0.2,
                            keep_logp=True)
    assert e.calls[-1][:2] == ("pixelcnn_generate", dict(temperature=1.0, top_k=0, want_logp=True, top_p=1.0, min_p=0.2, want_kept=True))
    assert k0.shape == lat0.shape and g.last_kept.shape == lat1.shape and g.last_kept.dtype == torch.int32


def test_wholebody_forwards_controls_and_sharded_equals_one_engine():
    from talkshow_b200.pipeline import WholeBody

    torch.set_grad_enabled(False)
    e = NucleusOracleEngine()
    wb = WholeBody(e)
    ck, vq = _ckpts("3d")
    wb.load(ck, vq, synth.face_checkpoint(0))
    B = 3
    mfcc = synth.synth_mfcc(B, 16, seed=16)
    wave = torch.randn(B, 16000 * 16 // 30, generator=torch.Generator().manual_seed(17))
    label = torch.tensor([0, 1, 3])
    noise = OS.reference_noise(18, 8, B)
    wb.generate(mfcc, wave, label, noise=noise)
    assert e.calls[-1] == ("body_generate", {}, False) and wb.last_kept is None
    one = wb.generate(mfcc, wave, label, noise=noise, temperature=0.9, top_p=0.7, min_p=0.01, keep_logp=True)
    assert e.calls[-1] == ("body_generate", dict(temperature=0.9, top_k=0, want_logp=True, top_p=0.7, min_p=0.01, want_kept=True), False)
    lp1, k1 = wb.last_logp, wb.last_kept
    assert k1.shape == (B, 4, 2) and (k1 >= 1).all()
    parts, lps, ks = [], [], []
    for r in range(2):
        parts.append(wb.generate_sharded(mfcc, wave, label, r, 2, noise_full=noise, gather=False, temperature=0.9, top_p=0.7,
                                         min_p=0.01, keep_logp=True))
        lps.append(wb.last_logp)
        ks.append(wb.last_kept)
    # the CPU stand-in's modules round differently at different batch sizes; the GPU test compares bit for bit
    assert (torch.cat(parts) - one).abs().max() <= 1e-5 and (torch.cat(lps) - lp1).abs().max() <= 1e-5
    assert torch.equal(torch.cat(ks), k1)
    wb.generate_sharded(mfcc, wave, label, 0, 1, noise_full=noise, top_p=0.6)
    assert e.calls[-1][1] == dict(temperature=1.0, top_k=0, want_logp=False, top_p=0.6, min_p=0.0, want_kept=False)


@pytest.mark.parametrize("kw", [dict(top_p=0.0), dict(top_p=-0.1), dict(top_p=1.5), dict(top_p=float("nan")), dict(top_p=1e-60),
                                dict(top_p="a"), dict(top_p=True), dict(min_p=-0.1), dict(min_p=1.01), dict(min_p=float("nan")),
                                dict(min_p=None)])
def test_invalid_controls_raise(kw):
    from talkshow_b200.engine import _controlled, check_sample_controls
    from talkshow_b200.pipeline import WholeBody

    args = dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0)
    args.update(kw)
    with pytest.raises(ValueError):
        check_sample_controls(**args)
    with pytest.raises(ValueError):
        _controlled(args["temperature"], args["top_k"], torch.ones(1), False, args["top_p"], args["min_p"])
    e = NucleusOracleEngine()
    g = _wrapper("6d", e)
    with pytest.raises(ValueError):
        g.generate(synth.synth_mfcc(1, 16, seed=1), torch.tensor([0]), **args)
    with pytest.raises(ValueError):
        WholeBody(e).generate(synth.synth_mfcc(1, 16, seed=1), torch.zeros(1, 8533), torch.tensor([0]), **args)
    assert e.calls == []


def _random_logits(scale, n=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 2048, generator=g) * scale


@pytest.mark.parametrize("scale", [0.5, 2.0, 8.0, 30.0])
@pytest.mark.parametrize("t,p", [(1.0, 0.9), (0.7, 0.5), (1.5, 0.99), (1.0, 0.05)])
def test_integer_rule_is_the_float64_nucleus(scale, t, p):
    """The keep set on integer masses is TopPLogitsWarper's (float64 sort and cumulative sum) wherever no boundary lies
    within 1e-6 of the threshold."""
    logits = _random_logits(scale, seed=int(scale * 10))
    keep, margin, _ = ON.keep_mask(logits, t, 0, p, 0.0, return_margin=True)
    ref = ON.top_p_reference(logits, t, p)
    clear = margin > 1e-6
    assert clear.sum() >= 20 and torch.equal(keep[clear], ref[clear])
    assert keep.gather(-1, logits.argmax(-1, keepdim=True)).all()                   # the most likely code is always kept
    # the kept mass reaches p, and without the boundary class it does not
    _, w, _ = ON.masses(logits, t)
    W = w.sum(-1).double()
    kept_mass = (w * keep).sum(-1).double()
    assert (kept_mass >= float(np.float32(p)) * W).all()
    low = torch.where(keep, logits, torch.full_like(logits, float("inf"))).min(-1, keepdim=True).values
    assert ((w * (logits > low)).sum(-1).double() < float(np.float32(p)) * W).all()


def test_permutation_invariance_and_ties():
    logits = _random_logits(4.0, n=8, seed=5)
    logits[:, 100:110] = logits[:, 7:8]                                   # a tie class of 11 codes
    logits[0, :] = 1.25                                                     # every code tied: all kept whatever p
    logits[1, 3] = 0.0
    logits[1, 4] = -0.0                                                     # -0 and +0 are one class
    perm = torch.randperm(2048, generator=torch.Generator().manual_seed(6))
    for t, k, p, m in [(1.0, 0, 0.9, 0.0), (0.8, 50, 0.6, 0.0), (1.2, 0, 0.95, 0.03), (1.0, 0, 1.0, 0.1)]:
        keep = ON.keep_mask(logits, t, k, p, m)
        assert torch.equal(ON.keep_mask(logits[:, perm], t, k, p, m), keep[:, perm])
        assert keep[0].all() or m > 0 or k > 0
        assert (keep[:, 100:110] == keep[:, 7:8]).all() and keep[1, 3] == keep[1, 4]
    assert ON.keep_mask(logits, 1.0, 0, 0.3, 0.0)[0].all()


def test_limits():
    """p -> 0 is greedy decoding, p = 1 with m = 0 is the draw of oracle_sampling, m = 1 keeps exactly the ties of the
    maximum, and a dropped code is never drawn."""
    g = torch.Generator().manual_seed(9)
    logits = torch.randn(16, 2048, generator=g) * 3.0
    logits[2, 500] = logits[2, 40] = logits[2].max() + 0.5                  # two codes tie for the maximum
    noise = torch.empty(16, 2048).exponential_(1, generator=g)
    code, kept = ON.draw(logits, noise, 1.0, 0, 1e-6, 0.0)
    greedy = OS.draw(logits, None, 0.0, 0)
    rows = torch.arange(16) != 2
    assert torch.equal(code[rows], greedy[rows]) and (kept[rows] == 1).all() and kept[2] == 2 and code[2] in (40, 500)
    for t, k in [(1.0, 0), (0.7, 0), (1.0, 33)]:
        code, kept = ON.draw(logits, noise, t, k, 1.0, 0.0)
        assert torch.equal(code, OS.draw(logits, noise, t, k)) and torch.equal(kept, OS.keep_mask(logits, k).sum(-1).to(torch.int32))
    keep = ON.keep_mask(logits, 0.9, 0, 1.0, 1.0)
    assert torch.equal(keep, logits == logits.max(-1, keepdim=True).values) and keep[2].sum() == 2
    for t, k, p, m in [(1.0, 0, 0.5, 0.0), (1.4, 20, 0.8, 0.05), (1.0, 0, 1.0, 0.3)]:
        keep = ON.keep_mask(logits, t, k, p, m)
        code, kept = ON.draw(logits, noise, t, k, p, m)
        assert keep.gather(-1, code[:, None]).all() and torch.equal(kept, keep.sum(-1).to(torch.int32))
        assert (keep & ~OS.keep_mask(logits, k)).sum() == 0                  # an intersection with the top-k set
    assert (ON.draw(logits, None, 0.0, 5, 0.5, 0.5)[1] == 1).all()          # greedy ignores the truncation
