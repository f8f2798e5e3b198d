"""GPU (-m gpu): ts_pixelcnn_score — the time-parallel teacher-forced GatedPixelCNN.forward with per-position
cross-entropy — against the CPU oracle, the reference goldens and the sampler, on both dense-kernel settings
(ts_set_tensor_cores 6: wgmma fp16-split, 0: FFMA)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import talkshow_oracle as O
from conftest import GOLDEN, ROOT, draw_noise
from talkshow_b200 import synth

sys.path.insert(0, GOLDEN)
from make_golden_prior_ce import bat_3d, bat_6d  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-4
MODES = [6, 0]


def _load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def _engine(ck, vq):
    from talkshow_b200.engine import Engine

    e = Engine(0)
    e.load_pixelcnn(ck["generator"])
    e.load_audioenc(ck["audioencoder"])
    e.load_vq(0, vq["g_body"])
    e.load_vq(1, vq["g_hand"])
    return e


@pytest.fixture(scope="module")
def eng(ckpts):
    e = _engine(ckpts["pixel"], ckpts["vq"])
    yield e
    torch.cuda.synchronize()
    e.close()


@pytest.fixture(scope="module")
def eng6():
    e = _engine(synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0))
    yield e
    torch.cuda.synchronize()
    e.close()


class _Mode:
    def __init__(self, e, mode):
        self.e, self.mode = e, mode

    def __enter__(self):
        self.e.set_tensor_cores(self.mode)

    def __exit__(self, *a):
        self.e.set_tensor_cores(6)


_REF = {}


def _case(sd, aenc, B, T, seed):
    """seeded inputs and the oracle's logits / NLL (cached across the two kernel settings)."""
    key = (id(sd), B, T, seed)
    if key not in _REF:
        g = torch.Generator().manual_seed(seed)
        codes = torch.randint(0, 2048, (B, T, 2), generator=g)
        label = torch.arange(B) % 4
        aud = O.audio_encoder(aenc, synth.synth_mfcc(B, 4 * T, seed=seed))
        logits = O.pixelcnn_forward(sd, codes, label, aud.unsqueeze(-1).repeat(1, 1, 1, 2))
        _REF[key] = (aud, label, codes, logits, F.cross_entropy(logits, codes, reduction="none"))
    return _REF[key]


def _check(e, sd, aenc, B, T, seed):
    aud, label, codes, ref_l, ref_nll = _case(sd, aenc, B, T, seed)
    nll, logits = e.pixelcnn_score(aud, label, codes, want_logits=True)
    err_l = (logits.cpu() - ref_l).abs().max().item()
    err_n = (nll.cpu() - ref_nll).abs().max().item()
    print("score B=%d T=%d: logits max-abs err %.3e, nll %.3e" % (B, T, err_l, err_n))
    assert nll.shape == (B, T, 2) and logits.shape == (B, 2048, T, 2)
    assert err_l <= TOL and err_n <= TOL
    # without logits: the same NLL
    assert torch.equal(e.pixelcnn_score(aud, label, codes), nll)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,T", [(3, 6), (1, 30), (64, 75), (100, 12)])
def test_score_vs_oracle(eng, ckpts, mode, B, T):
    """(64, 75) is the benchmark shape; B = 100 runs above the sampler's 64-sample tile."""
    with _Mode(eng, mode):
        _check(eng, ckpts["pixel"]["generator"], ckpts["pixel"]["audioencoder"], B, T, 100 + B + T)


@pytest.mark.parametrize("mode", MODES)
def test_score_reference_golden_b1_t30(eng, mode):
    """the teacher-forced logit rows the reference's GatedPixelCNN.forward produced (pixel_b1_t30.npz)."""
    gold = _load("pixel_b1_t30")
    with _Mode(eng, mode):
        nll, logits = eng.pixelcnn_score(torch.from_numpy(gold["audio"]), torch.tensor([0]), torch.from_numpy(gold["codes"]),
                                         want_logits=True)
    got = logits[0][:, gold["logit_rows"], :].cpu().numpy()
    assert np.abs(got - gold["logits"]).max() <= TOL


@pytest.mark.parametrize("mode", MODES)
def test_score_6d_geometry(eng6, mode):
    """dim 512 x 10 layers (convert_to_6d): the oracle, and the reference's logits of the prior_ce golden."""
    bp6 = synth.body_pixel_checkpoint_6d(0)
    gold = _load("prior_ce")
    with _Mode(eng6, mode):
        _check(eng6, bp6["generator"], bp6["audioencoder"], 3, 10, 7)
        bat = bat_6d()
        aud = eng6.audio_encode(bat["aud_feat"])
        _, logits = eng6.pixelcnn_score(aud, bat["speaker"] - 20, torch.from_numpy(gold["codes_6d"]), want_logits=True)
    got = logits[:, :, gold["logit_rows"], :].cpu().numpy()
    assert np.abs(got - gold["logits_6d"]).max() <= TOL


@pytest.mark.parametrize("mode", MODES)
def test_score_agrees_with_sampler(eng, ckpts, mode):
    """Score the codes the sampler drew: the logits at every drawn position agree, and the summed NLL equals the
    -log softmax the sampler's own logits give those codes."""
    B, T = 6, 20
    aud = O.audio_encoder(ckpts["pixel"]["audioencoder"], synth.synth_mfcc(B, 4 * T, seed=71))
    label = torch.tensor([0, 1, 2, 3, 0, 2])
    noise = draw_noise(2 * T, B, 72)
    with _Mode(eng, mode):
        codes, slog = eng.pixelcnn_generate(aud, label, noise, want_logits=True)      # slog [2T,B,2048]
        nll, logits = eng.pixelcnn_score(aud, label, codes, want_logits=True)
    slog = slog.view(T, 2, B, 2048).permute(2, 3, 0, 1)                              # -> [B,2048,T,2]
    assert (logits - slog).abs().max().item() <= TOL
    ref = -torch.log_softmax(slog.double(), 1).gather(1, codes.unsqueeze(1)).sum()
    assert abs(nll.double().sum().item() - ref.item()) <= 1e-3 * abs(ref.item())


def test_score_launches_do_not_grow_with_T(eng):
    """Time-parallel: one call issues the same kernels for 30 rows as for 75 (the sampler's chain issues stages per row)."""
    g = torch.Generator().manual_seed(5)
    counts = []
    for T in (30, 75):
        aud = torch.randn(4, 256, T, generator=g).cuda()
        label = torch.tensor([0, 1, 2, 3]).cuda()
        codes = torch.randint(0, 2048, (4, T, 2), generator=g).cuda()
        n0 = eng.launches
        eng.pixelcnn_score(aud, label, codes)
        counts.append(eng.launches - n0)
    assert counts[0] == counts[1] and counts[0] > 0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("key", ["3d", "6d"])
def test_evaluate_reference_ce_loss(eng, eng6, key, mode):
    """s2g_body_pixel.evaluate on the CUDA engine reproduces the reference's ce_loss (prior_ce.npz): within 1e-5 on the
    FFMA kernel.  The tensor core's fp32 accumulation truncates toward zero, which shrinks every layer's output a little;
    the mean NLL of these sharp synthetic priors (about 15) comes out 1-2e-5 low, hence 2.5e-5 on the wgmma kernel."""
    import types

    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    gold = _load("prior_ce")
    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Data.pose.convert_to_6d = key == "6d"
    cfg.Model.vq_path = ""
    g = TrainWrapper(types.SimpleNamespace(gpu=0, infer=False), cfg, engine=eng if key == "3d" else eng6)
    bat = bat_3d() if key == "3d" else bat_6d()
    with _Mode(g.engine, mode):
        out, losses = g.evaluate(bat)
    print("evaluate %s (mode %d): ce_loss %.7f (reference %.7f)" % (key, mode, losses["ce_loss"], float(gold["ce_" + key])))
    assert out is None and abs(losses["ce_loss"] - float(gold["ce_" + key])) <= (1e-5 if mode == 0 else 2.5e-5)
    assert np.array_equal(g.last_nll.shape, gold["codes_" + key].shape)
    # mismatched audio / pose lengths
    with pytest.raises(ValueError):
        g.evaluate(dict(bat, aud_feat=bat["aud_feat"][:, :, :80]))


def test_score_errors(eng):
    from talkshow_b200.engine import Engine

    L, s = eng.L, C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(1 << 16, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    assert L.ts_pixelcnn_score(eng.h, p, p, p, p, None, 0, 5, s) == 1        # TS_ERR_INVALID
    assert L.ts_pixelcnn_score(eng.h, p, p, p, p, None, 2, 0, s) == 1
    assert L.ts_pixelcnn_score(eng.h, p, p, p, p, None, -1, 5, s) == 1
    e = Engine(0)
    try:
        assert L.ts_pixelcnn_score(e.h, p, p, p, p, None, 1, 5, s) == 2      # TS_ERR_NOT_LOADED
        with pytest.raises(RuntimeError):
            e.pixelcnn_score(torch.zeros(1, 256, 5), torch.tensor([0]), torch.zeros(1, 5, 2, dtype=torch.int64))
    finally:
        e.close()
