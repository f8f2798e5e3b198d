"""CPU (-m "not gpu"): seeded sampling of the body prior.

The numpy Philox4x32-10 of tests/oracle_seeded.py against the published Random123 known-answer vectors; the layout of the
seeded noise (a clip's block depends only on its seed and the absolute row); its distribution; and the host layer (seed
helpers, validation, wrappers and sharded generation) on an oracle-backed stand-in engine that builds the seeded noise with
the numpy oracle."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle_engine import OracleEngine
from talkshow_b200 import synth

sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_seeded as OS  # noqa: E402


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(ctr, key, want):
    assert OS.philox4x32_10(ctr, key).tolist() == want


def test_contract_mapping():
    """code n of draw (r, c) is output n >> 9 of counter (n & 511, r, c, 0) under key (seed lo, seed hi)"""
    seed = -0x123456789ABCDEF          # negative: its 64 bits
    lo, hi = OS.seed_key(seed)
    assert (hi << 32 | lo) == seed & 0xFFFFFFFFFFFFFFFF
    u = OS.uniforms(seed, 5, 1)
    for n in (0, 1, 255, 256, 511, 512, 1023, 1536, 2047):
        x = int(OS.philox4x32_10([n & 511, 5, 1, 0], [lo, hi])[n >> 9])
        assert u[n] == ((x >> 8) | 1) * 2.0 ** -24
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)            # exact in fp32
    assert u.min() >= 2.0 ** -24 and u.max() <= 1 - 2.0 ** -24


def test_noise_layout():
    seeds = [11, -3, 2 ** 62, 7]
    full = OS.noise(seeds, 9)
    # a T0 call is the tail of a longer call (rows keyed absolutely)
    assert np.array_equal(OS.noise(seeds, 5, T0=4), full[8:])
    # a clip's block depends only on its seed: not on B or the clip's place in the batch
    for b, s in enumerate(seeds):
        assert np.array_equal(OS.noise([s], 9)[:, 0], full[:, b])
    assert np.array_equal(OS.noise([5, 11, 9], 9)[:, 1], full[:, 0])
    # different seeds, rows and columns give different noise
    assert not np.array_equal(full[:, 0], full[:, 3]) and not np.array_equal(full[0], full[1]) and not np.array_equal(full[0], full[2])
    assert np.isfinite(full).all() and (full > 0).all()


def test_distribution_is_exp1():
    from scipy import stats

    q = OS.noise([2024, 2025, 2026, 2027], 30).astype(np.float64).ravel()             # 4 clips x 60 draws x 2048
    ks = stats.kstest(q, "expon")
    assert ks.pvalue > 0.01, ks
    assert abs(q.mean() - 1) < 0.01 and abs(q.var() - 1) < 0.02, (q.mean(), q.var())
    # the uniforms are uniform on the odd multiples of 2^-24 (no bias at either end)
    u = OS.uniforms_block([99], 30).ravel()
    assert stats.kstest(u, "uniform").pvalue > 0.01


def test_seed_helpers():
    from talkshow_b200.engine import check_seeds, clip_seeds, resolve_clip_seeds

    assert clip_seeds(5, 3).tolist() == [5, 6, 7] and clip_seeds(5, 3).dtype == torch.int64
    assert clip_seeds(2 ** 63 - 1, 2).tolist() == [2 ** 63 - 1, -2 ** 63]                  # wraps to int64 bits
    assert clip_seeds(-1, 2).tolist() == [-1, 0]
    assert check_seeds([1, 2 ** 64 - 1], 2).tolist() == [1, -1]
    assert check_seeds(np.array([3, 4]), 2).tolist() == [3, 4]
    t = torch.tensor([9, 8], dtype=torch.int64)
    assert check_seeds(t, 2) is t
    assert torch.equal(resolve_clip_seeds(10, 2), clip_seeds(10, 2)) and resolve_clip_seeds(None, 4) is None
    assert torch.equal(resolve_clip_seeds([4, 5], 2), torch.tensor([4, 5]))
    for bad in (torch.tensor([1, 2], dtype=torch.int32), torch.zeros(2, 1, dtype=torch.int64), torch.tensor([1.0, 2.0]),
                [1, 2, 3], [1, 2.5], [True, 1], "ab", np.array([1.0, 2.0]), 3.5):
        with pytest.raises(ValueError):
            check_seeds(bad, 2)
    for bad in (True, 2.0, [1]):
        with pytest.raises(ValueError):
            resolve_clip_seeds(bad, 2)


def test_engine_validation_before_any_call():
    from talkshow_b200.engine import _controlled

    assert _controlled(1.0, 0, None, False, seeds=torch.zeros(1, dtype=torch.int64)) is False
    assert _controlled(0.0, 0, None, False) is True                                   # greedy needs neither
    with pytest.raises(ValueError):
        _controlled(1.0, 0, torch.ones(1), False, seeds=torch.zeros(1, dtype=torch.int64))   # both
    with pytest.raises(ValueError):
        _controlled(0.7, 0, None, False)                                              # neither while sampling


def test_host_only_engine_refuses_seeded_entry_points():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    e.load_pixelcnn(synth.pixelcnn_state(0))
    L, h, n = e.L, e.h, None
    for name, args in (("ts_sampler_noise", (h, n, n, 2, 3, 0, n)),
                       ("ts_pixelcnn_sample_seeded", (h, n, n, n, n, n, 1, 2, n, 0, n, n)),
                       ("ts_body_sample_seeded", (h, n, n, n, n, n, 1, 8, n, n))):
        assert getattr(L, name)(*args) != 0 and b"host-only" in L.ts_last_error(h), name
    e.close()


class SeededOracleEngine(OracleEngine):
    """OracleEngine plus ``seeds=`` on pixelcnn_generate / body_generate: the seeded noise is built by the numpy oracle
    (rows keyed from T0) and the call is answered like an explicit-noise call.  Every call is recorded in ``calls``."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []

    def pixelcnn_generate(self, aud, label, noise, T=None, pre_latents=None, want_logits=False, seeds=None):
        T0 = 0 if pre_latents is None else pre_latents.shape[1]
        T = aud.shape[2] - T0 if T is None else T
        self.calls.append(("pixelcnn_generate", None if seeds is None else seeds.tolist(), T0, noise is None))
        if seeds is not None:
            noise = torch.from_numpy(OS.noise(seeds.tolist(), T, T0))
        return super().pixelcnn_generate(aud, label, noise, T=T, pre_latents=pre_latents)

    def body_generate(self, mfcc, label, noise, want_codes=True, seeds=None):
        self.calls.append(("body_generate", None if seeds is None else seeds.tolist(), 0, noise is None))
        if seeds is not None:
            noise = torch.from_numpy(OS.noise(seeds.tolist(), self.latent_rows(mfcc.shape[2])))
        return super().body_generate(mfcc, label, noise, want_codes)


def _wrapper(engine):
    import types

    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Model.vq_path = ""
    g = TrainWrapper(types.SimpleNamespace(gpu=0, infer=True), cfg, engine=engine)
    g.load_state_dict(synth.body_pixel_checkpoint(0))
    g.load_vq_state_dict(synth.body_vq_checkpoint(0))
    g.noise_device = "cpu"
    return g


def test_wrapper_forwards_clip_seeds():
    torch.set_grad_enabled(False)
    e = SeededOracleEngine()
    g = _wrapper(e)
    B = 3
    mfcc = synth.synth_mfcc(B, 16, seed=4)
    label = torch.tensor([0, 1, 2])
    out = g.generate(mfcc, label, clip_seeds=40)
    assert e.calls[-1] == ("body_generate", [40, 41, 42], 0, True)                   # seed + b, no noise drawn
    # equals the explicit call on the oracle's seeded noise
    ref = g.generate(mfcc, label, noise_fn=lambda T, B_: torch.from_numpy(OS.noise([40, 41, 42], T)))
    assert torch.equal(out, ref) and e.calls[-1][3] is False
    g.generate(mfcc, label, clip_seeds=[7, -1, 2 ** 63])
    assert e.calls[-1][1] == [7, -1, -2 ** 63]
    g.generate(mfcc, label, clip_seeds=torch.tensor([1, 2, 3]))
    assert e.calls[-1][1] == [1, 2, 3]
    with pytest.raises(ValueError):
        g.generate(mfcc, label, noise_fn=lambda T, B_: None, clip_seeds=1)
    with pytest.raises(ValueError):
        g.infer(mfcc.transpose(1, 2), 0, label, B, noise_fn=lambda T, B_: None, clip_seeds=1)
    with pytest.raises(ValueError):
        g.infer_on_audio(mfcc[0].transpose(0, 1).numpy(), B=1, noise_fn=lambda T, B_: None, clip_seeds=1)
    for bad in ([1, 2], 1.5, torch.tensor([1, 2, 3], dtype=torch.int32)):
        with pytest.raises(ValueError):
            g.generate(mfcc, label, clip_seeds=bad)


def test_infer_chunks_keyed_from_T0():
    """the continuity path's second chunk gets the same seeds with its rows keyed after the prefix"""
    torch.set_grad_enabled(False)
    e = SeededOracleEngine()
    g = _wrapper(e)
    B = 2
    feat = synth.synth_mfcc(B, 32, seed=6).transpose(1, 2)                            # [B,M,64]
    label = torch.tensor([1])
    lat0, aud0, _, _ = g.infer(feat[:, :16], 0, label, B, clip_seeds=9)
    lat1, _, b1, _ = g.infer(feat[:, 16:], 0, label, B, lat0, aud0, clip_seeds=9)
    assert e.calls[-2] == ("pixelcnn_generate", [9, 10], 0, True) and e.calls[-1] == ("pixelcnn_generate", [9, 10], 4, True)
    ref1, _, rb1, _ = g.infer(feat[:, 16:], 0, label, B, lat0, aud0,
                              noise_fn=lambda T, B_: torch.from_numpy(OS.noise([9, 10], T, T0=4)))
    assert torch.equal(lat1, ref1) and torch.equal(b1, rb1)


def test_wholebody_and_sharded_with_clip_seeds():
    from talkshow_b200.pipeline import WholeBody

    torch.set_grad_enabled(False)
    e = SeededOracleEngine()
    wb = WholeBody(e)
    wb.load(synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), synth.face_checkpoint(0))
    B = 5
    mfcc = synth.synth_mfcc(B, 16, seed=26)
    wave = torch.randn(B, 16000 * 16 // 30, generator=torch.Generator().manual_seed(27))
    label = torch.tensor([0, 1, 3, 2, 0])
    one = wb.generate(mfcc, wave, label, clip_seeds=100)
    assert e.calls[-1] == ("body_generate", list(range(100, 105)), 0, True)
    for world in (1, 2, 3):
        parts = []
        for r in range(world):
            parts.append(wb.generate_sharded(mfcc, wave, label, r, world, gather=False, clip_seeds=100, seed=5))
        # the CPU stand-in's modules round differently at different batch sizes; the GPU test compares bit for bit
        assert (torch.cat(parts) - one).abs().max() <= 1e-5, world
    # rank r passes the seeds of its shard
    from talkshow_b200.pipeline import shard_range

    for r in range(3):
        wb.generate_sharded(mfcc, wave, label, r, 3, gather=False, clip_seeds=100)
        lo, hi = shard_range(B, r, 3)
        assert e.calls[-1] == ("body_generate", list(range(100 + lo, 100 + hi)), 0, True)
    with pytest.raises(ValueError):
        wb.generate(mfcc, wave, label, noise=torch.ones(8, B, 2048), clip_seeds=1)
    with pytest.raises(ValueError):
        wb.generate_sharded(mfcc, wave, label, 0, 2, noise_full=torch.ones(8, B, 2048), clip_seeds=1)
