"""CPU (-m "not gpu"): held-out scoring of a face / VQ / prior trio, pinned to the reference's own modules and get_loss
(tests/golden/eval_losses.npz, written by tests/golden/make_golden_eval.py) for a 3-D and a convert_to_6d trio.

The oracle restatement (tests/oracle_eval.py) is checked against the fixture; the wrappers' evaluate() and
WholeBody.evaluate run on an oracle-backed stand-in engine, so their host logic (c_index, body / hand split, target
assembly, ids, shape checks, loss reductions) is the same Python the GPU tests run on the CUDA engine."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import oracle_eval as OE
from conftest import GOLDEN, ROOT
from talkshow_b200 import synth
from talkshow_b200.data_utils.lower_body import c_index_3d, c_index_6d

sys.path.insert(0, GOLDEN)
from make_golden_eval import bat_3d, bat_6d, input_fingerprint  # noqa: E402

KEYS = ["3d", "6d"]


def trio(key):
    if key == "3d":
        return synth.face_checkpoint(0), synth.body_vq_checkpoint(0), synth.body_pixel_checkpoint(0), bat_3d()
    return synth.face_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0), synth.body_pixel_checkpoint_6d(0), bat_6d()


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "eval_losses.npz"))


def gold_losses(gold, key):
    return dict(zip([str(n) for n in gold["loss_names"]], gold["losses_" + key].tolist()))


def face_bat(bat):
    """The face wrapper's batch: its 'aud_feat' is the waveform [B,1,N]."""
    return {"aud_feat": bat["wave"][:, None, :], "poses": bat["poses"], "expression": bat["expression"],
            "speaker": bat["speaker"]}


def _cfg(name, six):
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", name + ".json"))
    cfg.Data.pose.convert_to_6d = six
    cfg.Model.vq_path = ""
    return cfg


def wrappers(key, engine):
    from talkshow_b200.nets import s2g_body_pixel, s2g_body_vq, s2g_face

    face, vq, bp, bat = trio(key)
    six = key == "6d"
    a = types.SimpleNamespace(gpu=0, infer=False)
    wf = s2g_face(a, _cfg("face", six), engine=engine)
    wf.load_state_dict(face)
    wv = s2g_body_vq(a, _cfg("body_vq", six), engine=engine)
    wv.load_state_dict(vq)
    wp = s2g_body_pixel(a, _cfg("body_pixel", six), engine=engine)
    wp.load_vq_state_dict(vq)
    wp.load_state_dict(bp)
    return wf, wv, wp, bat


def close(a, b, rel):
    return abs(a - b) <= rel * max(abs(b), 1e-30)


@pytest.mark.parametrize("key", KEYS)
def test_oracle_matches_reference(gold, key):
    torch.set_grad_enabled(False)
    face, vq, bp, bat = trio(key)
    assert np.allclose(gold["in_fp_" + key], input_fingerprint(bat), rtol=1e-12, atol=0)
    assert np.allclose(gold["fp_" + key], [list(synth.fingerprint(c).values()) for c in (face, vq, bp)], rtol=1e-12, atol=0)
    want = gold_losses(gold, key)
    stride = int(gold["stride"])
    # face: the oracle's wav2vec2 restatement vs the reference's HF module, fp32 both
    gt = torch.cat([bat["poses"].permute(0, 2, 1), bat["expression"].permute(0, 2, 1)], 2)
    idv = torch.nn.functional.one_hot(bat["speaker"] - 20, 4).float()
    pred, clip = OE.face_eval(face["generator"], bat["wave"], idv, gt)
    assert np.abs(pred[:, ::stride].numpy() - gold["pred_" + key]).max() <= 1e-4
    mse, exp = OE.face_get_loss(pred, gt)
    assert close(mse, want["MSELoss"], 1e-5) and close(exp, want["exp_loss"], 1e-5)
    assert np.allclose(clip.numpy(), gold["clip_face_" + key], rtol=1e-5, atol=0)
    # VQ pair: codes exact, recon within the existing VQ bar, losses and per-clip sums
    six = key == "6d"
    gtp = bat["poses"][:, c_index_6d if six else c_index_3d, :].permute(0, 2, 1)
    nb = 78 if six else 39
    for name, sd, part in (("b", vq["g_body"], gtp[..., :nb]), ("h", vq["g_hand"], gtp[..., nb:])):
        idx, recon, clip, e_q = OE.vq_eval(sd, part.contiguous())
        assert np.array_equal(idx.numpy(), gold["codes_%s_%s" % (name, key)])
        assert np.abs(recon[:, ::stride].numpy() - gold["recon_%s_%s" % (name, key)]).max() <= 1e-4
        rec, vel = OE.vq_get_loss(recon, part)
        assert close(rec, want[name + "rec_loss"], 1e-5) and close(vel, want[name + "velocity_loss"], 1e-5)
        assert np.allclose(clip.numpy(), gold["clip_%s_%s" % (name, key)], rtol=1e-5, atol=0)
        assert close(e_q, float(gold["e_q_%s_%s" % (name, key)]), 1e-5)


@pytest.mark.parametrize("key", KEYS)
def test_wrapper_evaluates_on_oracle_engine(gold, key):
    torch.set_grad_enabled(False)
    wf, wv, wp, bat = wrappers(key, OE.EvalOracleEngine())
    want = gold_losses(gold, key)
    out, lf = wf.evaluate(face_bat(bat))
    assert out is None and list(lf) == ["MSELoss", "exp_loss"]
    out, lv = wv.evaluate(bat)
    assert out is None and list(lv) == ["brec_loss", "bvelocity_loss", "hrec_loss", "hvelocity_loss"]
    _, lp = wp.evaluate(bat)
    for k, v in dict(lf, **lv, **lp).items():
        # evaluate() sums per clip in fp64, the reference takes torch.mean over fp32: a few fp32 ulps apart
        assert close(v, want[k], 1e-5), (k, v, want[k])
    B, nf = bat["poses"].shape[0], bat["poses"].shape[2]
    per = wv.last_losses
    assert set(per) == {"brec_loss", "bvelocity_loss", "be_q_loss", "hrec_loss", "hvelocity_loss", "he_q_loss"}
    for name in "bh":
        assert close(float(per[name + "rec_loss"].mean()), lv[name + "rec_loss"], 1e-12)
        # per-clip commitment terms average to the reference's commitment_cost * mse(z, e)
        assert close(float(per[name + "e_q_loss"].mean()), float(gold["e_q_%s_%s" % (name, key)]), 1e-5)
        assert per[name + "e_q_loss"].shape == (B,)
    assert tuple(wv.last_codes.shape) == (B, nf // 4, 2)
    assert np.array_equal(wv.last_codes[..., 0].numpy(), gold["codes_b_" + key])
    assert set(wf.last_losses) == {"MSELoss", "exp_loss"} and wf.last_losses["MSELoss"].shape == (B,)


@pytest.mark.parametrize("key", KEYS)
def test_whole_body_evaluate_on_oracle_engine(gold, key):
    from talkshow_b200.pipeline import WholeBody

    torch.set_grad_enabled(False)
    face, vq, bp, bat = trio(key)
    wb = WholeBody(OE.EvalOracleEngine())
    wb.load(bp, vq, face)
    out, losses = wb.evaluate(bat)
    assert out is None
    assert list(losses) == ["MSELoss", "exp_loss", "brec_loss", "bvelocity_loss", "hrec_loss", "hvelocity_loss", "ce_loss"]
    want = gold_losses(gold, key)
    for k, v in losses.items():
        assert close(v, want[k], 1e-5), (k, v, want[k])
    # the same numbers as the three wrapper calls
    wf, wv, wp, _ = wrappers(key, OE.EvalOracleEngine())
    merged = dict(wf.evaluate(face_bat(bat))[1], **wv.evaluate(bat)[1], **wp.evaluate(bat)[1])
    assert losses == merged
    assert tuple(wb.last_nll.shape) == (bat["poses"].shape[0], bat["poses"].shape[2] // 4, 2)


def test_evaluate_rejects_bad_batches():
    torch.set_grad_enabled(False)
    from talkshow_b200.pipeline import WholeBody

    wf, wv, wp, bat = wrappers("3d", OE.EvalOracleEngine())
    face, vq, bp, _ = trio("3d")
    wb = WholeBody(OE.EvalOracleEngine())
    wb.load(bp, vq, face)
    cut = {k: (v[:, :, :118] if k in ("poses", "expression") else v) for k, v in bat.items()}   # F % 4 != 0
    with pytest.raises(ValueError):
        wv.evaluate(cut)
    with pytest.raises(ValueError):
        wb.evaluate(dict(cut, aud_feat=bat["aud_feat"][:, :, :118]))
    with pytest.raises(ValueError):                                     # 80 feature frames -> 20 rows vs 30 code rows
        wb.evaluate(dict(bat, aud_feat=bat["aud_feat"][:, :, :80]))
    with pytest.raises(ValueError):                                     # 6-D pose block under the 3-D geometry
        wv.evaluate(dict(bat, poses=torch.cat([bat["poses"], bat["poses"]], 1)))
    with pytest.raises(ValueError):
        wb.evaluate(dict(bat, poses=torch.cat([bat["poses"], bat["poses"]], 1)))
    with pytest.raises(ValueError):                                     # expression frames differ from the pose frames
        wf.evaluate(dict(face_bat(bat), expression=bat["expression"][:, :, :100]))
    with pytest.raises(ValueError):                                     # 3-D pose block under the 6-D trio
        wv6 = wrappers("6d", OE.EvalOracleEngine())[1]
        wv6.evaluate(bat)
