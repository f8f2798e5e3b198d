"""CPU (-m "not gpu"): the body prior's cross-entropy on ground-truth motion (s2g_body_pixel.evaluate), pinned to the
reference's own training-step loss (tests/golden/prior_ce.npz, written by tests/golden/make_golden_prior_ce.py from
s2g_body_pixel.__call__ with the generator and audio encoder in eval mode).

``prior_ce`` restates the forward half of nets/smplx_body_pixel.py:183-216 with the oracle's modules; the wrapper's
evaluate() is driven on an oracle-backed stand-in engine, so the host logic (c_index, body / hand split, speaker ids,
row check, loss reduction) is the same Python the GPU test runs on the CUDA engine."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import talkshow_oracle as O
from conftest import GOLDEN, ROOT
from oracle_engine import OracleEngine
from talkshow_b200 import synth

sys.path.insert(0, GOLDEN)
from make_golden_prior_ce import bat_3d, bat_6d  # noqa: E402


def prior_ce(ckpt, vq_ckpt, bat, c_index, n_body):
    """s2g_body_pixel.__call__ (:183-216) up to F.cross_entropy, eval mode: (ce_loss, codes [B,T,2], logits [B,2048,T,2])."""
    aud = bat["aud_feat"].float()
    label = bat["speaker"] - 20
    gt = bat["poses"].float()[:, c_index, :].permute(0, 2, 1)
    _, body = O.vq_encode(vq_ckpt["g_body"], gt[..., :n_body])
    _, hand = O.vq_encode(vq_ckpt["g_hand"], gt[..., n_body:])
    lat = torch.stack([body, hand], -1)
    audio = O.audio_encoder(ckpt["audioencoder"], aud).unsqueeze(-1).repeat(1, 1, 1, 2)
    logits = O.pixelcnn_forward(ckpt["generator"], lat, label, audio)
    lg = logits.permute(0, 2, 3, 1).contiguous()
    return F.cross_entropy(lg.view(-1, lg.shape[-1]), lat.view(-1)).item(), lat, logits


class ScoringOracleEngine(OracleEngine):
    """OracleEngine plus Engine.pixelcnn_score answered by the oracle forward and F.cross_entropy."""

    def pixelcnn_score(self, aud, label, codes, want_logits=False):
        B, _, T = aud.shape
        label = label.reshape(-1).to(torch.int64)
        if label.numel() == 1 and B > 1:
            label = label.expand(B)
        logits = O.pixelcnn_forward(self.sd["pixelcnn"], codes, label, aud.float().unsqueeze(-1).repeat(1, 1, 1, 2))
        nll = F.cross_entropy(logits, codes, reduction="none")
        return (nll, logits) if want_logits else nll


def _case(key):
    if key == "3d":
        return synth.body_pixel_checkpoint(0), synth.body_vq_checkpoint(0), bat_3d(), False
    return synth.body_pixel_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0), bat_6d(), True


def _wrapper(key, engine):
    from talkshow_b200.nets.smplx_body_pixel import TrainWrapper
    from talkshow_b200.trainer.config import load_JsonConfig

    ck, vq, bat, six = _case(key)
    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    cfg.Data.pose.convert_to_6d = six
    cfg.Model.vq_path = ""
    g = TrainWrapper(types.SimpleNamespace(gpu=0, infer=False), cfg, engine=engine)
    g.load_vq_state_dict(vq)
    g.load_state_dict(ck)
    return g, bat


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "prior_ce.npz"))


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_prior_ce_oracle_matches_reference(gold, key):
    torch.set_grad_enabled(False)
    ck, vq, bat, six = _case(key)
    assert np.allclose(gold["fp_" + key], list(synth.fingerprint(ck).values()), rtol=1e-12, atol=0)
    assert np.allclose(gold["in_fp_" + key], [float(bat["aud_feat"].double().sum()), float(bat["poses"].double().sum())],
                       rtol=1e-12, atol=0)
    from talkshow_b200.data_utils.lower_body import c_index_3d, c_index_6d

    ce, lat, logits = prior_ce(ck, vq, bat, c_index_6d if six else c_index_3d, 78 if six else 39)
    assert np.array_equal(lat.numpy(), gold["codes_" + key])
    assert np.abs(logits[:, :, gold["logit_rows"], :].numpy() - gold["logits_" + key]).max() <= 1e-4
    assert abs(ce - float(gold["ce_" + key])) <= 1e-6


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_evaluate_on_oracle_engine(gold, key):
    torch.set_grad_enabled(False)
    g, bat = _wrapper(key, ScoringOracleEngine())
    out, losses = g.evaluate(bat)
    assert out is None and set(losses) == {"ce_loss"}
    # the reference reduces in fp32 inside F.cross_entropy, evaluate() averages the per-position NLL in fp64: the two
    # orders differ by a few fp32 ulps of a loss near 15, so the bar is relative
    assert abs(losses["ce_loss"] - float(gold["ce_" + key])) <= 1e-6 * float(gold["ce_" + key])
    assert g.last_nll.shape == tuple(gold["codes_" + key].shape)


def test_evaluate_rejects_row_mismatch():
    """Audio and pose clips whose latent rows differ: the reference fails in the prior's concatenation."""
    torch.set_grad_enabled(False)
    g, bat = _wrapper("3d", ScoringOracleEngine())
    bad = dict(bat, aud_feat=bat["aud_feat"][:, :, :80])          # 80 feature frames -> 20 rows vs 22 code rows
    with pytest.raises(ValueError):
        g.evaluate(bad)
