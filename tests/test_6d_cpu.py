"""CPU (-m "not gpu"): the convert_to_6d whole-body path.  The oracle's 6-D pieces (tests/oracle_6d.py) against the
fixtures the unmodified reference wrote (tests/golden/make_golden_6d.py: face_6d.npz, vq_6d.npz, demo_flow_6d.npz); the 6-D
wrappers, scripts/demo.py and pipeline.WholeBody driven on an oracle-backed engine against the same fixtures; checkpoint
geometry checks on a host-only engine (weights are packed, nothing executes)."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

import oracle_6d as O6
import talkshow_oracle as O
from conftest import GOLDEN, ROOT, draw_noise, noise_fp
from oracle_engine import OracleEngine
from talkshow_b200 import synth

sys.path.insert(0, GOLDEN)
from make_golden_6d import poses_6d  # noqa: E402


class OracleEngine6D(OracleEngine):
    """OracleEngine plus the convert_to_6d surface of Engine: face_dim, the identity-free face, the 6-D assembly."""

    @property
    def face_dim(self):
        sd = self.sd.get("face")
        return 0 if sd is None else int(sd["final_out.0.weight"].shape[0] + sd["final_out.1.weight"].shape[0])

    def face_forward(self, wave, id_onehot, frame):
        wave = wave.float().reshape(wave.shape[0], -1)
        idv = id_onehot.float()
        if idv.shape[0] == 1 and wave.shape[0] > 1:
            idv = idv.expand(wave.shape[0], -1)
        return O6.face_forward(self.sd["face"], wave, idv, frame)

    def body_generate(self, mfcc, label, noise, want_codes=True):
        # one sample at a time, as the reference's demo loop runs them: ATen's CPU convs round differently per batch size,
        # and the 6-D -> axis-angle conversion magnifies those last bits where the Gram-Schmidt step is ill-conditioned
        label = label.reshape(-1).expand(mfcc.shape[0])
        outs = [super(OracleEngine6D, self).body_generate(mfcc[b:b + 1], label[b:b + 1], noise[:, b:b + 1], want_codes)
                for b in range(mfcc.shape[0])]
        return (torch.cat([o[0] for o in outs]) if want_codes else None), torch.cat([o[1] for o in outs])

    def assemble_pose(self, face, body, stand=False):
        if face.shape[2] == 103:
            return super().assemble_pose(face, body, stand)
        return torch.stack([O6.assemble_pose_6d(face[b], body[b], stand) for b in range(face.shape[0])])


def _load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def _cfg(name, six):
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", name + ".json"))
    cfg.Data.pose.convert_to_6d = six
    return cfg


def _args():
    return types.SimpleNamespace(gpu=0, infer=True)      # resolve_device(0) -> cuda:0 (no CUDA call); the engine is injected


@pytest.fixture(scope="module")
def ck6():
    torch.set_grad_enabled(False)
    return {"face": synth.face_checkpoint_6d(0), "vq": synth.body_vq_checkpoint_6d(0), "pixel": synth.body_pixel_checkpoint_6d(0)}


@pytest.fixture()
def shared(monkeypatch):
    import talkshow_b200.nets.base as base

    eng = OracleEngine6D()
    monkeypatch.setattr(base, "_ENGINES", {0: eng})
    return eng


# ---- the oracle against the reference ---------------------------------------------------------------------------------

def test_face_6d_schema_is_the_identity_free_net(ck6):
    sd = ck6["face"]["generator"]
    assert "audio_middle.id_mlp.weight" not in sd and not any("residual_layer" in k for k in sd)
    assert tuple(sd["audio_middle.first_net.conv_layers.0.conv.weight"].shape) == (256, 256, 3)
    assert tuple(sd["final_out.0.weight"].shape) == (6, 64, 1) and tuple(sd["final_out.1.weight"].shape) == (100, 256, 1)
    assert set(synth.face_schema()) - set(synth.face_schema(identity=False, jaw_dim=6)) == {
        "audio_middle.id_mlp.weight", "audio_middle.id_mlp.bias", "audio_middle.first_net.conv_layers.0.residual_layer.0.weight",
        "audio_middle.first_net.conv_layers.0.residual_layer.0.bias"}


def test_oracle_face_6d_matches_reference(ck6):
    g = _load("face_6d")
    assert np.allclose(g["fp"], list(synth.fingerprint(ck6["face"]).values()), rtol=1e-12, atol=0)
    sd = ck6["face"]["generator"]
    out = O6.face_forward(sd, synth.synth_wave(1, 64000), torch.zeros(1, 4), 120).numpy()
    assert out.shape == g["out_4s"].shape == (1, 120, 106)
    assert np.abs(out - g["out_4s"]).max() <= 1e-6
    ids = torch.nn.functional.one_hot(torch.tensor(g["ids_10s"]), 4).float()
    wave = synth.synth_wave(2, 160000, seed=int(g["wave_seed_10s"]))
    out = O6.face_forward(sd, wave, ids, 300).numpy()
    err = max(np.abs(out[:, ::int(g["out_10s_stride"])] - g["out_10s"]).max(), np.abs(out[:, :8] - g["out_10s_head"]).max())
    assert err <= 1e-6, err
    assert np.array_equal(out, O6.face_forward(sd, wave, torch.zeros(2, 4), 300).numpy())       # id is ignored


def test_oracle_vq_6d_matches_reference(ck6):
    g = _load("vq_6d")
    assert np.allclose(g["fp_vq"], list(synth.fingerprint(ck6["vq"]).values()), rtol=1e-12, atol=0)
    ib, ih, out = O6.body_vq_roundtrip_6d(ck6["vq"], poses_6d(2, 88, seed=int(g["pose_seed"])))
    assert np.array_equal(ib.numpy(), g["idx_body"]) and np.array_equal(ih.numpy(), g["idx_hand"])
    assert out.shape == g["out"].shape == (88, 516)
    assert np.abs(out.numpy() - g["out"]).max() <= 1e-6
    outc = O6.body_vq_continuity_6d(ck6["vq"], poses_6d(2, 300, seed=int(g["pose_seed_cont"]))).numpy()
    assert outc.shape == (300, 516)
    assert np.abs(outc[::int(g["out_cont_stride"])] - g["out_cont"]).max() <= 1e-6
    assert np.abs(outc[56:64] - g["out_cont_seam"]).max() <= 1e-6


def _demo_inputs(tmp_path, g):
    from scipy.io import wavfile

    sec = int(g["seconds"])
    x = (synth.synth_wave(1, 16000 * sec, seed=int(g["wave_seed"]))[0].numpy() * 20000).astype(np.int16)
    wav = str(tmp_path / "clip six.wav")
    wavfile.write(wav, 16000, x)
    return wav


def _reference_face_pass_rng():
    from talkshow_b200.nets.smplx_face import hf_layerdrop_uses_torch_rng

    if hf_layerdrop_uses_torch_rng():
        for _ in range(12):
            torch.rand([])


def _same_stream(g, T):
    from talkshow_b200.nets.smplx_face import hf_layerdrop_uses_torch_rng

    return (np.allclose(g["noise_fp"], noise_fp(draw_noise(2 * T, 1, int(g["seed"]))), rtol=0, atol=1e-9)
            and hf_layerdrop_uses_torch_rng() == bool(g["hf_torch_layerdrop"]))


def test_oracle_demo_flow_6d_matches_reference(ck6, tmp_path):
    """scripts/demo.py:infer of the reference for a convert_to_6d config, restated sample by sample on the oracle."""
    from talkshow_b200.data_utils.utils import load_wav, mfcc_from_wave

    g = _load("demo_flow_6d")
    assert np.allclose(g["fp_face"], list(synth.fingerprint(ck6["face"]).values()), rtol=1e-12, atol=0)
    assert np.allclose(g["fp_body"], list(synth.fingerprint(ck6["pixel"]).values()), rtol=1e-12, atol=0)
    audio, sr = load_wav(_demo_inputs(tmp_path, g))
    frame = int(g["frame"])
    face = O6.face_forward(ck6["face"]["generator"], audio, torch.zeros(1, 4), frame)[0]
    mfcc = torch.from_numpy(mfcc_from_wave(audio, sr, sr=22000, fps=30).T.copy())[None]
    T = O.latent_rows(mfcc.shape[2])
    if not _same_stream(g, T):
        pytest.skip("this host's CPU generator / transformers draw a different stream than the fixture's")
    seed, spk = int(g["seed"]), int(g["speaker"])
    for stand, n, key in ((False, int(g["num_sample"]), "saved"), (True, 1, "saved_stand")):
        torch.manual_seed(seed)
        _reference_face_pass_rng()
        rows = []
        for i in range(n):
            noise = torch.stack([torch.empty(1, 2048).exponential_(1) for _ in range(2 * T)])
            codes, body = O.body_generate(ck6["pixel"], ck6["vq"], mfcc, torch.tensor([spk]), noise=noise, window=18)
            if not stand:
                assert np.array_equal(codes[0].numpy(), g["codes"][i])
            rows.append(O6.assemble_pose_6d(face, body[0], stand))
        assert np.abs(torch.cat(rows).numpy() - g[key]).max() <= 1e-5, key


# ---- host layer on an oracle-backed engine against the reference ---------------------------------------------------

def test_face_wrapper_6d(ck6, shared):
    from talkshow_b200.nets import s2g_face

    g = _load("face_6d")
    w = s2g_face(_args(), _cfg("face", True))
    assert w.each_dim == [6, 144, 180, 100] and w.dim_list == [0, 6, 18, 150, 330]
    w.load_state_dict({"generator": {"module." + k: v for k, v in ck6["face"]["generator"].items()}})
    out = w.infer_on_audio(synth.synth_wave(1, 64000)[:, None, :])
    assert out.shape == (1, 120, 106) and np.abs(out - g["out_4s"]).max() <= 1e-6
    out_id = w.infer_on_audio(synth.synth_wave(1, 64000)[:, None, :], id=torch.tensor([3]))
    assert np.array_equal(out, out_id)
    assert tuple(w.generate(synth.synth_wave(2, 24000, seed=5)[:, None, :], 45).shape) == (2, 45, 106)


def test_body_vq_wrapper_6d(ck6, shared):
    from talkshow_b200.nets import s2g_body_vq

    g = _load("vq_6d")
    w = s2g_body_vq(_args(), _cfg("body_vq", True))
    assert w.each_dim[1:3] == [78, 180]
    w.load_state_dict(ck6["vq"])
    out = w.infer_on_audio(torch.zeros(2, 64, 88), initial_pose=poses_6d(2, 88, seed=int(g["pose_seed"])), fps=30)
    assert out.shape == (88, 516) and np.abs(out - g["out"]).max() <= 1e-6
    ib, ih = w.encode(poses_6d(2, 88, seed=int(g["pose_seed"])))
    assert np.array_equal(ib.numpy(), g["idx_body"]) and np.array_equal(ih.numpy(), g["idx_hand"])
    outc = w.infer_on_audio(None, initial_pose=poses_6d(2, 300, seed=int(g["pose_seed_cont"])), continuity=True, fps=30)
    assert outc.shape == (300, 516)
    assert np.abs(outc[::int(g["out_cont_stride"])] - g["out_cont"]).max() <= 1e-6
    assert np.abs(outc[56:64] - g["out_cont_seam"]).max() <= 1e-6


def test_demo_flow_6d_on_the_oracle_engine(ck6, tmp_path, monkeypatch, shared):
    """talkshow_b200.scripts.demo with a convert_to_6d copy of config/body_pixel.json, 6-D checkpoint files and the
    reference's command line writes the (num_sample*F, 265) .npy the reference's scripts/demo.py writes."""
    from talkshow_b200.scripts import demo

    g = _load("demo_flow_6d")
    wav = _demo_inputs(tmp_path, g)
    for name, ck in (("body6.pth", ck6["pixel"]), ("face6.pth", ck6["face"]), ("vq6.pth", ck6["vq"])):
        torch.save({"generator": ck}, str(tmp_path / name))
    cfg_json = json.load(open(os.path.join(ROOT, "config", "body_pixel.json")))
    cfg_json["Data"]["pose"]["convert_to_6d"] = True
    cfg_json["Model"]["vq_path"] = str(tmp_path / "vq6.pth")
    json.dump(cfg_json, open(str(tmp_path / "cfg6.json"), "w"))
    import talkshow_b200.nets.base as base
    monkeypatch.setattr(base, "resolve_device", lambda gpu: torch.device("cpu"))
    for mod in ("smplx_body_pixel", "smplx_face"):
        monkeypatch.setattr(__import__("talkshow_b200.nets." + mod, fromlist=["x"]), "resolve_device", base.resolve_device)
    orig_init = demo.init_model

    def init_cpu_noise(name, path, a, c):
        w = orig_init(name, path, a, c)
        w.noise_device = "cpu"
        return w

    monkeypatch.setattr(demo, "init_model", init_cpu_noise)
    monkeypatch.chdir(tmp_path)
    seed, nsamp, frame = int(g["seed"]), int(g["num_sample"]), int(g["frame"])
    argv = ["--config_file", str(tmp_path / "cfg6.json"), "--infer", "--audio_file", wav, "--id", str(int(g["speaker"])),
            "--body_model_path", str(tmp_path / "body6.pth"), "--face_model_path", str(tmp_path / "face6.pth")]
    torch.manual_seed(seed)
    result_list, _ = demo.main(argv + ["--num_sample", str(nsamp)])
    saved = np.load(str(tmp_path / "visualise" / "video" / str(g["log_name"]) / "clip six.npy"))
    assert saved.shape == (nsamp * frame, 265)
    assert shared.face_dim == 106 and shared.vq_dim(0) == 78
    mfcc_T = O.latent_rows(frame)            # 3 s: 90 feature frames at 30 fps
    if not _same_stream(g, mfcc_T):
        pytest.skip("this host's CPU generator / transformers draw a different stream than the fixture's")
    assert np.abs(saved - g["saved"]).max() <= 1e-5
    torch.manual_seed(seed)
    demo.main(argv + ["--num_sample", "1", "--stand"])
    saved = np.load(str(tmp_path / "visualise" / "video" / str(g["log_name"]) / "clip six.npy"))
    assert np.abs(saved - g["saved_stand"]).max() <= 1e-5


def test_whole_body_6d_host_logic(ck6):
    """pipeline.WholeBody with 6-D checkpoints: face (106) + body (258) -> 6-D assembly, sharding does not change it."""
    from talkshow_b200.pipeline import WholeBody

    wb = WholeBody(OracleEngine6D())
    wb.load(ck6["pixel"], ck6["vq"], ck6["face"])
    assert wb.e2 is None
    B = 3
    wave = synth.synth_wave(B, 16000 + 800, seed=12)                    # 31 face frames, 28 body frames
    mfcc = synth.synth_mfcc(B, 30, seed=13)
    label = torch.tensor([1, 3, 0])
    noise = draw_noise(2 * O.latent_rows(30), B, 5)
    got = wb.generate(mfcc, wave, label, noise=noise)
    face = O6.face_forward(ck6["face"]["generator"], wave, torch.zeros(B, 4), 31)
    body = torch.cat([O.body_generate(ck6["pixel"], ck6["vq"], mfcc[b:b + 1], label[b:b + 1], noise=noise[:, b:b + 1], window=18)[1]
                      for b in range(B)])
    assert face.shape[2] == 106 and body.shape[1:] == (28, 258)
    ref = torch.stack([O6.assemble_pose_6d(face[b], body[b]) for b in range(B)])
    assert got.shape == (B, 31, 265) and torch.equal(got, ref)
    # each rank runs its contiguous shard with the shard's slice of the full-batch noise; ATen's CPU face convs round
    # differently per batch size, so each shard is checked against the oracle run at that shard's batch
    for r, (lo, hi) in enumerate(((0, 2), (2, 3))):
        part = wb.generate_sharded(mfcc, wave, label, r, 2, noise_full=noise, gather=False)
        f = O6.face_forward(ck6["face"]["generator"], wave[lo:hi], torch.zeros(hi - lo, 4), 31)
        assert torch.equal(part, torch.stack([O6.assemble_pose_6d(f[b - lo], body[b]) for b in range(lo, hi)]))


# ---- checkpoint geometry on the real library (host-only engine) ------------------------------------------------------

def test_face_geometry_checks(ck6):
    from talkshow_b200.engine import Engine
    from talkshow_b200.nets import s2g_face

    e = Engine(-148)
    assert e.face_dim == 0
    e.load_face(ck6["face"]["generator"])
    assert e.face_dim == 106
    e.load_face(synth.face_checkpoint(0)["generator"])
    assert e.face_dim == 103
    w6 = s2g_face(_args(), _cfg("face", True), engine=e)
    with pytest.raises(RuntimeError, match="jaw 3"):
        w6.load_state_dict(synth.face_checkpoint(0))                 # 3-D face checkpoint under a 6-D config
    assert e.face_dim == 103                                         # refused before anything was loaded
    w3 = s2g_face(_args(), _cfg("face", False), engine=e)
    with pytest.raises(RuntimeError, match="jaw 6"):
        w3.load_state_dict(ck6["face"])                              # 6-D face checkpoint under a 3-D config
    # malformed identity-free checkpoints: the error names the offending tensor, the loaded net stays as it was
    bad = dict(synth.face_checkpoint(0)["generator"])
    bad.pop("audio_middle.id_mlp.weight")
    bad.pop("audio_middle.id_mlp.bias")
    bad.pop("audio_middle.first_net.conv_layers.0.residual_layer.0.weight")
    with pytest.raises(RuntimeError, match=r"first_net\.conv_layers\.0\.conv\.weight"):
        e.load_face(bad)                                             # 320-channel layer 0 without id_mlp
    bad = dict(ck6["face"]["generator"])
    bad["audio_middle.first_net.conv_layers.0.residual_layer.0.weight"] = torch.zeros(256, 256, 3)
    with pytest.raises(RuntimeError, match=r"residual_layer\.0\.weight"):
        e.load_face(bad)
    assert e.face_dim == 103                                         # still the last net that loaded
    e.close()


def test_vq_geometry_checks(ck6):
    from talkshow_b200.engine import Engine
    from talkshow_b200.nets import s2g_body_vq

    e = Engine(-148)
    with pytest.raises(RuntimeError, match="78, 180"):
        s2g_body_vq(_args(), _cfg("body_vq", True), engine=e).load_state_dict(synth.body_vq_checkpoint(0))
    with pytest.raises(RuntimeError, match="39, 90"):
        s2g_body_vq(_args(), _cfg("body_vq", False), engine=e).load_state_dict(ck6["vq"])
    cfg = _cfg("body_vq", True)
    cfg.Model.composition = False
    with pytest.raises(NotImplementedError):
        s2g_body_vq(_args(), cfg, engine=e)
    w = s2g_body_vq(_args(), _cfg("body_vq", True), engine=e)
    w.config.Data.pose.normalization = True
    with pytest.raises(NotImplementedError):
        w.infer_on_audio(None, initial_pose=poses_6d(1, 88, seed=1))
    e.close()


def test_assemble_pose_rejects_other_layouts():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    for fd, bd in ((103, 258), (106, 129), (104, 129), (106, 256)):
        with pytest.raises(ValueError):
            e.assemble_pose(torch.zeros(1, 4, fd), torch.zeros(1, 4, bd))
    with pytest.raises(ValueError):
        e.assemble_pose(torch.zeros(2, 4, 106), torch.zeros(1, 4, 258))      # batch sizes differ
    e.close()
