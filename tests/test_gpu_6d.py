"""GPU (-m gpu): the convert_to_6d whole-body path on the CUDA engine — the identity-free 6-D face net on both kernel
settings, the fused 6-D pose assembly (ts_assemble_pose6d), pipeline.WholeBody with 6-D checkpoints, and the 6-D demo flow
against the file the reference's scripts/demo.py writes (tests/golden/demo_flow_6d.npz)."""
import json
import math
import os

import numpy as np
import pytest
import torch

import oracle_6d as O6
from conftest import GOLDEN, ROOT, draw_noise, noise_fp
from talkshow_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ck6():
    torch.set_grad_enabled(False)
    return {"face": synth.face_checkpoint_6d(0), "vq": synth.body_vq_checkpoint_6d(0), "pixel": synth.body_pixel_checkpoint_6d(0)}


def _engine(face_sd, tc=True):
    from talkshow_b200.engine import Engine

    e = Engine(0)
    if not tc:
        e.set_tensor_cores(0)
    e.load_face(face_sd)
    return e


def _joint_mask(mask55):
    """[n,55] per-joint mask -> [n,265] column mask (joints are the 3-column groups below column 165)."""
    cols = torch.zeros(mask55.shape[0], 265, dtype=torch.bool)
    cols[:, :165] = mask55[:, :, None].expand(-1, -1, 3).reshape(-1, 165)
    return cols


def _aa_close(got, ref, tol_rot=5e-3, tol=1e-4):
    """got vs ref [..., 265]: the columns that are not axis-angle joints (lower-pose constants, expression) within tol; the
    joint columns, which come out of the fp32 6-D -> axis-angle conversion, within tol_rot, leaving out joints whose
    rotation lies within 0.1 rad of pi.  Two fp32 evaluations of that conversion do not agree to 1e-4: small quaternion
    components are square roots of cancellation residues, and nearly parallel or short 6-D columns magnify rounding in the
    Gram-Schmidt step.  On 2M random normal 6-D inputs the oracle's fp32 result is up to 1.5e-3 from its own float64
    evaluation away from pi (tests/test_gpu_parity.py::test_rot6d_to_axis_angle uses 1e-3 on 4k inputs); the bar here
    covers the ~1M joints of a 64 x 10 s batch.  The fused assembly's exact equality with ts_rot6d_to_axis_angle followed by
    ts_assemble_pose is checked bit for bit separately.  Returns (joint error, other-column error, joints left out)."""
    got, ref = got.reshape(-1, 265).double(), ref.reshape(-1, 265).double()
    near_pi = ref[:, :165].reshape(-1, 55, 3).norm(dim=-1) > math.pi - 0.1
    joints = _joint_mask(torch.ones_like(near_pi))
    d = (got - ref).abs()
    err_other = d[~joints].max().item()
    err_rot = (d * _joint_mask(~near_pi)).max().item()
    print("6-D poses: joints max-abs %.3e, other columns %.3e, %d of %d joints near pi left out"
          % (err_rot, err_other, int(near_pi.sum()), near_pi.numel()))
    assert err_other <= tol and err_rot <= tol_rot, (err_rot, err_other, int(near_pi.sum()))
    return err_rot, err_other, int(near_pi.sum())


@pytest.mark.parametrize("B,sec", [(1, 4), (64, 10), (1, 53)])
def test_face_6d_matches_oracle(ck6, B, sec):
    sd = ck6["face"]["generator"]
    wave = synth.synth_wave(B, 16000 * sec, seed=B + sec)
    frame = sec * 30
    ids = torch.nn.functional.one_hot(torch.arange(B) % 4, 4).float()
    sel = sorted({0, B // 2, B - 1})               # the oracle runs on these clips alone (per-clip independence is checked too)
    ref = O6.face_forward(sd, wave[sel], ids[sel], frame)
    for tc in (True, False):
        e = _engine(sd, tc)
        assert e.face_dim == 106
        got = e.face_forward(wave, ids, frame)
        assert got.shape == (B, frame, 106) and torch.isfinite(got).all()
        err = (got[sel].cpu() - ref).abs().max().item()
        print("6-D face B=%d %d s tensor cores %s: max-abs err vs oracle %.3e" % (B, sec, tc, err))
        assert err <= 1e-4, (tc, err)
        torch.cuda.synchronize()
        e.close()


def test_face_6d_matches_reference_golden(ck6):
    g = np.load(os.path.join(GOLDEN, "face_6d.npz"))
    e = _engine(ck6["face"]["generator"])
    out = e.face_forward(synth.synth_wave(1, 64000), torch.zeros(1, 4), 120).cpu().numpy()
    assert np.abs(out - g["out_4s"]).max() <= 1e-4
    ids = torch.nn.functional.one_hot(torch.tensor(g["ids_10s"]), 4).float()
    out = e.face_forward(synth.synth_wave(2, 160000, seed=int(g["wave_seed_10s"])), ids, 300).cpu().numpy()
    assert np.abs(out[:, ::int(g["out_10s_stride"])] - g["out_10s"]).max() <= 1e-4
    assert np.abs(out[:, :8] - g["out_10s_head"]).max() <= 1e-4
    torch.cuda.synchronize()
    e.close()


def test_identity_free_net_drops_two_launches(ck6):
    """The identity-free net runs neither the id-column kernel nor the layer-0 residual conv; everything else is shared."""
    wave = synth.synth_wave(2, 32000, seed=3)
    counts = {}
    for key, sd in (("3d", synth.face_checkpoint(0)["generator"]), ("6d", ck6["face"]["generator"])):
        e = _engine(sd)
        e.face_forward(wave, torch.zeros(2, 4), 60)
        n0 = e.launches
        e.face_forward(wave, torch.zeros(2, 4), 60)
        counts[key] = e.launches - n0
        torch.cuda.synchronize()
        e.close()
    assert counts["3d"] - counts["6d"] == 2, counts


def test_reload_3d_after_6d_is_bit_identical(ck6):
    face3 = synth.face_checkpoint(0)["generator"]
    wave = synth.synth_wave(2, 48000, seed=4)
    ids = torch.nn.functional.one_hot(torch.tensor([1, 3]), 4).float()
    e = _engine(ck6["face"]["generator"])
    e.face_forward(wave, ids, 90)
    e.load_face(face3)
    assert e.face_dim == 103
    again = e.face_forward(wave, ids, 90)
    fresh = _engine(face3)
    assert torch.equal(again, fresh.face_forward(wave, ids, 90))
    torch.cuda.synchronize()
    e.close()
    fresh.close()


@pytest.mark.parametrize("Fb", [7, 13])
@pytest.mark.parametrize("stand", [False, True])
def test_assemble_pose6d_equals_convert_then_assemble(stand, Fb):
    from talkshow_b200.engine import Engine

    e = Engine(0)
    B, Ff = 3, 10
    g = torch.Generator().manual_seed(Fb + 10 * int(stand))
    face = torch.randn(B, Ff, 106, generator=g).cuda()
    body = torch.randn(B, Fb, 258, generator=g).cuda()
    fused = e.assemble_pose(face, body, stand)
    jaw = e.rot6d_to_axis_angle(face[..., :6])
    body_aa = e.rot6d_to_axis_angle(body.reshape(B, Fb, 43, 6)).reshape(B, Fb, 129)
    two_step = e.assemble_pose(torch.cat([jaw, face[..., 6:]], -1), body_aa, stand)
    assert fused.shape == (B, Ff, 265) and torch.equal(fused, two_step)
    ref = torch.stack([O6.assemble_pose_6d(face[b].cpu(), body[b].cpu(), stand) for b in range(B)])
    _aa_close(fused.cpu(), ref)
    torch.cuda.synchronize()
    e.close()


def _noise(T, B, seed):
    return torch.empty(2 * T, B, 2048).exponential_(1, generator=torch.Generator().manual_seed(seed))


def test_whole_body_6d_matches_oracle_composition(ck6):
    """WholeBody.generate at 64 x 10 s == the oracle's demo.py assembly of the engine's own face and body outputs."""
    from talkshow_b200.engine import Engine
    from talkshow_b200.pipeline import WholeBody

    e = Engine(0)
    wb = WholeBody(e)
    wb.load(ck6["pixel"], ck6["vq"], ck6["face"])
    assert wb.e2 is None and e.face_dim == 106 and e.vq_dim(0) + e.vq_dim(1) == 258
    B, M = 64, 300
    wave = synth.synth_wave(B, 160000, seed=21).cuda()
    mfcc = synth.synth_mfcc(B, M, seed=22).cuda()
    label = (torch.arange(B) % 4).cuda()
    noise = _noise(e.latent_rows(M), B, 23).cuda()
    got = wb.generate(mfcc, wave, label, noise=noise)
    face = e.face_forward(wave, torch.zeros(B, 4), 300)
    _, body = e.body_generate(mfcc, label, noise, want_codes=False)
    assert got.shape == (B, 300, 265) and body.shape == (B, 300, 258)
    ref = torch.stack([O6.assemble_pose_6d(face[b].cpu(), body[b].cpu()) for b in range(B)])
    _aa_close(got.cpu(), ref)
    host = wb.generate_host(mfcc.cpu().pin_memory(), wave.cpu().pin_memory(), label.cpu().pin_memory(), noise=noise)
    assert torch.equal(host, got.cpu())
    torch.cuda.synchronize()
    e.close()


def test_sharded_6d_equals_one_engine(ck6):
    """world 2 as two engines on one device: the shards' poses rebuild the one-engine batch."""
    from talkshow_b200.engine import Engine
    from talkshow_b200.pipeline import WholeBody

    wbs = []
    for _ in range(2):
        wb = WholeBody(Engine(0))
        wb.load(ck6["pixel"], ck6["vq"], ck6["face"])
        wbs.append(wb)
    B, M = 5, 120
    mfcc, wave = synth.synth_mfcc(B, M, seed=31), synth.synth_wave(B, 64000, seed=32)
    label = torch.arange(B) % 4
    noise = _noise(wbs[0].e.latent_rows(M), B, 33).cuda()
    parts = [wbs[r].generate_sharded(mfcc, wave, label, r, 2, noise_full=noise, gather=False) for r in range(2)]
    assert [p.shape[0] for p in parts] == [3, 2]
    got = torch.cat(parts, 0)
    ref = wbs[0].generate(mfcc.cuda(), wave.cuda(), label.cuda(), noise=noise)
    print("6-D sharded (world 2) vs one engine: identical %s, max-abs diff %.3e" % (torch.equal(got, ref), (got - ref).abs().max().item()))
    assert torch.equal(got, ref)
    torch.cuda.synchronize()
    for wb in wbs:
        wb.e.close()


def test_demo_flow_6d_matches_reference(ck6, tmp_path, monkeypatch):
    """talkshow_b200.scripts.demo with a convert_to_6d config and 6-D checkpoint files reproduces the .npy the reference's
    scripts/demo.py writes under the same seed (tests/golden/make_golden_6d.py): codes exactly; poses within 1e-4 outside the
    axis-angle joints, and within the conversion's bar (see _aa_close) on the joints away from pi."""
    from scipy.io import wavfile

    from talkshow_b200.nets.smplx_face import hf_layerdrop_uses_torch_rng
    from talkshow_b200.scripts import demo
    from talkshow_b200.trainer.config import load_JsonConfig
    from talkshow_b200.trainer.options import parse_args

    g = np.load(os.path.join(GOLDEN, "demo_flow_6d.npz"))
    sec, nsamp, spk, seed = int(g["seconds"]), int(g["num_sample"]), int(g["speaker"]), int(g["seed"])
    x = (synth.synth_wave(1, 16000 * sec, seed=int(g["wave_seed"]))[0].numpy() * 20000).astype(np.int16)
    wav = str(tmp_path / "clip six.wav")
    wavfile.write(wav, 16000, x)
    for name, ck in (("body6.pth", ck6["pixel"]), ("face6.pth", ck6["face"]), ("vq6.pth", ck6["vq"])):
        torch.save({"generator": ck}, str(tmp_path / name))
    cfg_json = json.load(open(os.path.join(ROOT, "config", "body_pixel.json")))
    cfg_json["Data"]["pose"]["convert_to_6d"] = True
    cfg_json["Model"]["vq_path"] = str(tmp_path / "vq6.pth")
    json.dump(cfg_json, open(str(tmp_path / "cfg6.json"), "w"))
    import talkshow_b200.nets.base as base
    from talkshow_b200.engine import Engine
    monkeypatch.setattr(base, "_ENGINES", {0: Engine(0)})              # a fresh engine for this flow
    orig_init = demo.init_model

    def init_host_noise(name, path, a, c):
        w = orig_init(name, path, a, c)
        w.noise_device = "cpu"                 # the CPU reference's sampling stream
        w.device_mfcc = False                  # the host torchaudio features the reference computed
        return w

    monkeypatch.setattr(demo, "init_model", init_host_noise)
    monkeypatch.chdir(tmp_path)
    argv = ["--config_file", str(tmp_path / "cfg6.json"), "--infer", "--audio_file", wav, "--id", str(spk),
            "--body_model_path", str(tmp_path / "body6.pth"), "--face_model_path", str(tmp_path / "face6.pth")]
    args = parse_args().parse_args(argv + ["--num_sample", str(nsamp)])
    config = load_JsonConfig(str(tmp_path / "cfg6.json"))
    g_body = demo.init_model(args.body_model_name, args.body_model_path, args, config)
    g_face = demo.init_model(args.face_model_name, args.face_model_path, args, config)
    torch.manual_seed(seed)
    result_list, _ = demo.infer(g_body, g_face, None, None, config, args)
    saved = np.load(str(tmp_path / "visualise" / "video" / str(g["log_name"]) / "clip six.npy"))
    frame = int(g["frame"])
    assert saved.shape == (nsamp * frame, 265)
    T = g["codes"].shape[1]
    if not (np.allclose(g["noise_fp"], noise_fp(draw_noise(2 * T, 1, seed)), rtol=0, atol=1e-9)
            and hf_layerdrop_uses_torch_rng() == bool(g["hf_torch_layerdrop"])):
        pytest.skip("this host's CPU generator / transformers draw a different stream than the fixture's")
    assert np.array_equal(g_body.last_codes.cpu().numpy(), g["codes"])
    _aa_close(torch.from_numpy(saved), torch.from_numpy(g["saved"]))
    args1 = parse_args().parse_args(argv + ["--num_sample", "1", "--stand"])
    torch.manual_seed(seed)
    res, _ = demo.infer(g_body, g_face, None, None, config, args1, save=False)
    _aa_close(res[0].cpu(), torch.from_numpy(g["saved_stand"]))
