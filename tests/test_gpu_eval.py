"""GPU (-m gpu): held-out scoring — ts_vq_score, ts_face_score and WholeBody.evaluate — on both dense-kernel settings
(ts_set_tensor_cores 6: wgmma fp16-split, 0: FFMA) and both geometries.

  - the forward outputs are the existing paths' bits: indices = vq_encode, recon = vq_decode(vq_encode(.)), pred =
    face_forward;
  - the per-clip sums agree with an fp64 restatement over the engine's own recon / pred (isolates the reductions);
  - the losses agree with the CPU oracle and the reference fixture (eval_losses.npz) within bars derived from the
    elementwise differences of the outputs they reduce;
  - WholeBody.evaluate equals the three wrapper calls with the VQ encode of the pair saved; repeated calls are
    bit-identical; generation is unchanged by an evaluate; bad arguments return error statuses."""
import ctypes as C
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
from make_golden_eval import bat_3d, bat_6d, synth_expression  # noqa: E402

pytestmark = pytest.mark.gpu
MODES = [6, 0]
SHAPES = [(64, 300), (1, 120), (3, 60)]


def trio(key):
    if key == "3d":
        return synth.face_checkpoint(0), synth.body_vq_checkpoint(0), synth.body_pixel_checkpoint(0)
    return synth.face_checkpoint_6d(0), synth.body_vq_checkpoint_6d(0), synth.body_pixel_checkpoint_6d(0)


@pytest.fixture(scope="module")
def wbs():
    from talkshow_b200.engine import Engine
    from talkshow_b200.pipeline import WholeBody

    out = {}
    for key in ("3d", "6d"):
        face, vq, bp = trio(key)
        wb = WholeBody(Engine(0), overlap_batch=0)
        wb.load(bp, vq, face)
        out[key] = wb
    yield out
    torch.cuda.synchronize()
    for wb in out.values():
        wb.close()
        wb.e.close()


class _Mode:
    def __init__(self, e, mode):
        self.e, self.mode = e, mode

    def __enter__(self):
        self.e.set_tensor_cores(self.mode)

    def __exit__(self, *a):
        self.e.set_tensor_cores(6)


def batch(key, B, nf, seed=5):
    """A trio batch of B clips x nf frames (poses [B,165|330,F], expression, wave, MFCC, speakers)."""
    poses = synth.synth_poses(B, nf, seed=seed)
    if key == "6d":
        poses = torch.cat([poses, synth.synth_poses(B, nf, seed=seed + 1)], 1)
    return {"wave": synth.synth_wave(B, -(-nf * 16000 // 30), seed=seed + 2), "aud_feat": synth.synth_mfcc(B, nf, seed=seed + 3),
            "poses": poses, "expression": synth_expression(B, nf, seed + 4), "speaker": 20 + torch.arange(B) % 4}


def split(key, poses):
    six = key == "6d"
    gt = poses[:, c_index_6d if six else c_index_3d, :].permute(0, 2, 1)
    nb = 78 if six else 39
    return gt[..., :nb].contiguous(), gt[..., nb:].contiguous()


def face_inputs(bat):
    gt = torch.cat([bat["poses"].permute(0, 2, 1), bat["expression"].permute(0, 2, 1)], 2).contiguous()
    return bat["wave"], torch.nn.functional.one_hot(bat["speaker"] - 20, 4).float(), gt


def rel_ok(got, want, rel):
    return torch.all((got - want).abs() <= rel * want.abs()).item()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,nf", SHAPES)
@pytest.mark.parametrize("key", ["3d", "6d"])
def test_vq_score_outputs_and_sums(wbs, key, B, nf, mode):
    e = wbs[key].e
    bat = batch(key, B, nf)
    with _Mode(e, mode):
        for w, part in enumerate(split(key, bat["poses"])):
            idx, clip, recon = e.vq_score(w, part, want_recon=True)
            assert torch.equal(idx, e.vq_encode(w, part))
            assert torch.equal(recon, e.vq_decode(w, idx).transpose(1, 2))
            # the reductions alone: fp64 over the engine's own recon
            r, g = recon.cpu(), part
            rec = (r - g).abs().double().sum((1, 2))
            vel = ((r[:, 1:] - r[:, :-1]) - (g[:, 1:] - g[:, :-1])).abs().double().sum((1, 2))
            c = clip.cpu()
            assert c.dtype == torch.float64 and c.shape == (B, 3)
            assert rel_ok(c[:, 0], rec, 1e-6) and rel_ok(c[:, 1], vel, 1e-6)
            # repeated calls, with and without recon: the same bits
            idx2, clip2, _ = e.vq_score(w, part)
            assert torch.equal(idx2, idx) and torch.equal(clip2, clip)
            if B * nf <= 360:
                # the commitment sums against the oracle's ||z - e||^2 (z of the oracle's fp32 encoder)
                _, _, oclip, _ = OE.vq_eval(wbs_sd(key, w), part)
                assert rel_ok(c[:, 2], oclip[:, 2], 1e-3)


def wbs_sd(key, w):
    return trio(key)[1]["g_hand" if w else "g_body"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,nf", SHAPES)
@pytest.mark.parametrize("key", ["3d", "6d"])
def test_face_score_outputs_and_sums(wbs, key, B, nf, mode):
    e = wbs[key].e
    wave, idv, gt = face_inputs(batch(key, B, nf))
    with _Mode(e, mode):
        clip, pred = e.face_score(wave, idv, gt, want_pred=True)
        assert torch.equal(pred, e.face_forward(wave, idv, nf))
        p = pred.cpu()
        l1 = (p[..., :6] - gt[..., :6]).abs().double().sum((1, 2))
        se = ((p[..., -100:] - gt[..., -100:]) ** 2).double().sum((1, 2))
        c = clip.cpu()
        assert c.dtype == torch.float64 and c.shape == (B, 2)
        assert rel_ok(c[:, 0], l1, 1e-6) and rel_ok(c[:, 1], se, 1e-6)
        clip2, _ = e.face_score(wave, idv, gt)
        assert torch.equal(clip2, clip)


_ORACLE = {}


def oracle_outputs(key, bat):
    """The oracle's pred / recon pair and its reference-style losses for the fixture batch (cached across modes)."""
    if key not in _ORACLE:
        face, vq, _ = trio(key)
        wave, idv, gt = face_inputs(bat)
        pred, _ = OE.face_eval(face["generator"], wave, idv, gt)
        out = {"pred": pred, "losses": dict(zip(("MSELoss", "exp_loss"), OE.face_get_loss(pred, gt)))}
        for name, w, part in zip("bh", (0, 1), split(key, bat["poses"])):
            _, recon, _, _ = OE.vq_eval(vq["g_hand" if w else "g_body"], part)
            out["recon_" + name] = recon
            out["losses"].update(zip((name + "rec_loss", name + "velocity_loss"), OE.vq_get_loss(recon, part)))
        _ORACLE[key] = out
    return _ORACLE[key]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("key", ["3d", "6d"])
def test_losses_vs_oracle_and_reference(wbs, key, mode):
    """|d mean|x|| <= max|dx| for the L1 terms (2 max|d recon| for the velocity term, whose differences take two frames);
    for the expression MSE, |mean(a^2) - mean(b^2)| <= max|a - b| * mean|a + b| with a, b the two residuals.  Against the
    reference the oracle's own distance to it (measured here) is added.  ce_loss: the prior scorer's documented bias
    (DESIGN §4), 5e-5 on losses near 15-20."""
    gold = np.load(os.path.join(GOLDEN, "eval_losses.npz"))
    want = dict(zip([str(n) for n in gold["loss_names"]], gold["losses_" + key].tolist()))
    bat = bat_3d() if key == "3d" else bat_6d()
    o = oracle_outputs(key, bat)
    wb = wbs[key]
    e = wb.e
    with _Mode(e, mode):
        _, losses = wb.evaluate(bat)
        wave, idv, gt = face_inputs(bat)
        _, pred = e.face_score(wave, idv, gt, want_pred=True)
        recon = {n: e.vq_score(w, part, want_recon=True)[2].cpu() for n, w, part in zip("bh", (0, 1), split(key, bat["poses"]))}
    pred = pred.cpu()
    dp = (pred - o["pred"]).abs().max().item()
    a, b = pred[..., -100:] - gt[..., -100:], o["pred"][..., -100:] - gt[..., -100:]
    bars = {"MSELoss": dp, "exp_loss": dp * (a + b).abs().double().mean().item(), "ce_loss": 5e-5}
    for n in "bh":
        dr = (recon[n] - o["recon_" + n]).abs().max().item()
        bars[n + "rec_loss"], bars[n + "velocity_loss"] = dr, 2 * dr
    for k, v in losses.items():
        slack = 1e-6 * abs(want[k])                                     # fp64 sum vs the reference's fp32 mean
        print("%s %s mode %d: %.7f (oracle %s, reference %.7f, bar %.2e)" % (key, k, mode, v, o["losses"].get(k), want[k], bars[k]))
        if k in o["losses"]:
            assert abs(v - o["losses"][k]) <= bars[k] + slack
            assert abs(v - want[k]) <= bars[k] + abs(o["losses"][k] - want[k]) + 2 * slack
        else:
            assert abs(v - want[k]) <= bars[k]


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_whole_body_equals_wrappers(wbs, key):
    """WholeBody.evaluate returns the three wrappers' dicts, bit for bit, and launches exactly the VQ encode of the
    pair fewer kernels (its codes come from the VQ score); a second call gives the same bits."""
    from talkshow_b200.nets import s2g_body_pixel, s2g_body_vq, s2g_face
    from talkshow_b200.trainer.config import load_JsonConfig

    wb = wbs[key]
    e = wb.e
    bat = batch(key, 3, 120, seed=17)

    def cfg(name):
        c = load_JsonConfig(os.path.join(ROOT, "config", name + ".json"))
        c.Data.pose.convert_to_6d = key == "6d"
        c.Model.vq_path = ""
        return c

    a = types.SimpleNamespace(gpu=0, infer=False)
    wf, wv, wp = s2g_face(a, cfg("face"), engine=e), s2g_body_vq(a, cfg("body_vq"), engine=e), s2g_body_pixel(a, cfg("body_pixel"), engine=e)
    n0 = e.launches
    _, losses = wb.evaluate(bat)
    n1 = e.launches
    fbat = {"aud_feat": bat["wave"][:, None, :], "poses": bat["poses"], "expression": bat["expression"], "speaker": bat["speaker"]}
    merged = dict(wf.evaluate(fbat)[1], **wv.evaluate(bat)[1], **wp.evaluate(bat)[1])
    n2 = e.launches
    for w, part in enumerate(split(key, bat["poses"])):
        e.vq_encode(w, part)
    n_enc = e.launches - n2
    torch.cuda.synchronize()
    assert losses == merged
    assert (n2 - n1) - (n1 - n0) == n_enc > 0
    last = {k: v.clone() for k, v in wb.last_losses.items()}
    assert wb.evaluate(bat)[1] == losses
    for k, v in wb.last_losses.items():
        assert torch.equal(v, last[k])
    assert torch.equal(wv.last_codes, torch.stack(split_codes(e, key, bat), -1))


def split_codes(e, key, bat):
    return [e.vq_encode(w, part) for w, part in enumerate(split(key, bat["poses"]))]


@pytest.mark.parametrize("key", ["3d", "6d"])
def test_generation_unchanged_by_evaluate(wbs, key):
    from talkshow_b200.nets.base import draw_sampler_noise

    wb = wbs[key]
    B, M = 2, 64
    mfcc = synth.synth_mfcc(B, M, seed=31).cuda()
    wave = synth.synth_wave(B, M * 16000 // 30, seed=32).cuda()
    label = torch.tensor([1, 3], device="cuda")
    noise = draw_sampler_noise(wb.e.latent_rows(M), B, torch.device("cuda"))
    before = wb.generate(mfcc, wave, label, noise=noise)
    wb.evaluate(batch(key, 2, 60, seed=33))
    after = wb.generate(mfcc, wave, label, noise=noise)
    torch.cuda.synchronize()
    assert torch.equal(before, after)


def test_score_errors(wbs):
    from talkshow_b200.engine import Engine

    e = wbs["3d"].e
    L, s = e.L, C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(1 << 20, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    assert L.ts_vq_score(e.h, 0, p, p, p, p, 1, 90, s) == 1             # TS_ERR_INVALID: F % 4 != 0
    assert L.ts_vq_score(e.h, 0, p, p, p, p, 0, 120, s) == 1
    assert L.ts_vq_score(e.h, 0, p, p, None, None, 1, 120, s) == 1      # clip_out missing
    assert L.ts_vq_score(e.h, 2, p, p, p, p, 1, 120, s) == 2            # TS_ERR_NOT_LOADED
    assert L.ts_face_score(e.h, p, p, p, 99, p, p, 1, 16000, 30, s) == 1   # gt without 100 expression columns
    assert L.ts_face_score(e.h, p, p, p, 103, p, p, 1, 100, 30, s) == 1    # too few samples
    assert L.ts_face_score(e.h, p, None, p, 103, p, p, 1, 16000, 30, s) == 1   # the identity net needs id
    assert L.ts_face_score(e.h, p, p, p, 103, p, None, 1, 16000, 30, s) == 1
    with pytest.raises(ValueError):
        e.vq_score(0, torch.zeros(1, 90, 39))
    with pytest.raises(ValueError):
        e.vq_score(0, torch.zeros(1, 120, 90))
    with pytest.raises(ValueError):
        e.face_score(torch.zeros(1, 16000), torch.zeros(1, 4), torch.zeros(1, 30, 99))
    e2 = Engine(0)
    try:
        assert L.ts_vq_score(e2.h, 0, p, p, p, p, 1, 120, s) == 2
        assert L.ts_face_score(e2.h, p, p, p, 103, p, p, 1, 16000, 30, s) == 2
    finally:
        e2.close()
