"""Generate the convert_to_6d fixtures by running the UNMODIFIED reference (a checkout named by $TALKSHOW_REFERENCE) on the
seeded synthetic 6-D checkpoints of talkshow_b200/synth.py.  Run on a host with that checkout:

    TALKSHOW_REFERENCE=/path/to/TalkSHOW python tests/golden/make_golden_6d.py

Writes, and leaves every other fixture as tests/golden/make_golden.py wrote it:
  face_6d.npz       s2g_face under a convert_to_6d config (identity=False, 6-D jaw head), eval / infer mode:
                    B = 1 at 4 s through infer_on_audio, B = 2 at 10 s through the generator with two different ids
                    (the identity-free net ignores them: the script checks that other ids give the same output);
  vq_6d.npz         s2g_body_vq.infer_on_audio round trip over the 6-D pose layout (c_index_6d, 78 + 180 channels),
                    plain and continuity=True (five 60-frame chunks);
  demo_flow_6d.npz  the .npy that scripts/demo.py:infer writes for a convert_to_6d config with 6-D face / pixel / VQ
                    checkpoints: num_sample 2, and the --stand variant with one sample, under a recorded seed.
"""
import importlib.machinery
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import torch  # noqa: E402

from make_golden import draw_noise, noise_fp  # noqa: E402
from ref_import import import_reference  # noqa: E402
from talkshow_b200 import synth  # noqa: E402

DEMO_SECONDS, DEMO_SAMPLES, DEMO_SPEAKER, DEMO_SEED, DEMO_WAVE_SEED = 3, 2, 1, 654, 43


def poses_6d(B, F, seed):
    """A [B,330,F] pose block in the 6-D layout: two axis-angle-scale blocks stacked (as make_golden_prior_ce.bat_6d)."""
    return torch.cat([synth.synth_poses(B, F, seed=seed), synth.synth_poses(B, F, seed=seed + 1)], 1)


def config_6d(load_JsonConfig, vq_path):
    cfg = load_JsonConfig("config/body_pixel.json")
    cfg.Data.pose.convert_to_6d = True
    cfg.Model.vq_path = vq_path
    return cfg


def main():
    cwd = os.getcwd()
    import_reference()
    REF_DIR = os.getcwd()
    import nets.smplx_body_vq as ref_vq
    import nets.smplx_face as ref_face
    from trainer.config import load_JsonConfig
    torch.set_grad_enabled(False)

    tmp = tempfile.mkdtemp()
    face6 = synth.face_checkpoint_6d(0)
    vq6 = synth.body_vq_checkpoint_6d(0)
    bp6 = synth.body_pixel_checkpoint_6d(0)
    vq6_path = os.path.join(tmp, "vq6.pth")
    torch.save({"generator": vq6}, vq6_path)
    cfg = config_6d(load_JsonConfig, vq6_path)
    a = types.SimpleNamespace(gpu="cpu", infer=True)

    # ---- face: identity-free net, 6-D jaw (nets/smplx_face.py:37-45,63-93) --------------------------------------------
    gf = ref_face.TrainWrapper(a, cfg)
    gf.generator.load_state_dict(face6["generator"], strict=True)
    assert not gf.generator.audio_middle.identity and gf.each_dim == [6, 144, 180, 100]
    assert gf.dim_list == [0, 6, 18, 150, 330]
    gf.generator.eval()
    wave = synth.synth_wave(1, 64000)
    o1 = gf.infer_on_audio(wave[:, None, :])                                          # (1,120,106), id=None
    wave2 = synth.synth_wave(2, 160000, seed=8)
    ids = torch.tensor([2, 0])
    o2 = gf.generator(wave2[:, None, :], None, torch.nn.functional.one_hot(ids, 4), time_steps=300)[0].numpy()   # (2,300,106)
    o2b = gf.generator(wave2[:, None, :], None, torch.nn.functional.one_hot(torch.tensor([3, 1]), 4), time_steps=300)[0].numpy()
    assert o1.shape == (1, 120, 106) and o2.shape == (2, 300, 106) and np.array_equal(o2, o2b)
    np.savez_compressed(os.path.join(HERE, "face_6d.npz"), out_4s=o1, out_10s=o2[:, ::4].copy(), out_10s_stride=4,
                        out_10s_head=o2[:, :8].copy(), ids_10s=ids.numpy(), wave_seed_10s=8,
                        fp=np.array(list(synth.fingerprint(face6).values())))
    print("face_6d", o1.shape, o2.shape, float(np.abs(o2).max()))

    # ---- VQ round trip over the 6-D layout (nets/smplx_body_vq.py:96-126, 208-295) ------------------------------------
    gv = ref_vq.TrainWrapper(a, cfg)
    gv.load_state_dict(vq6)
    assert gv.each_dim[1:3] == [78, 180]
    poses = poses_6d(2, 88, seed=621)
    outv = gv.infer_on_audio(torch.zeros(2, 64, 88), initial_pose=poses, fps=30)              # (88, 516)
    gt = poses[:, gv.c_index].permute(0, 2, 1)
    _, ib = gv.g_body.encode(gt_poses=gt[..., :78])
    _, ih = gv.g_hand.encode(gt_poses=gt[..., 78:])
    outc = gv.infer_on_audio(torch.zeros(2, 64, 300), initial_pose=poses_6d(2, 300, seed=623), continuity=True, fps=30)  # (300, 516)
    assert outv.shape == (88, 516) and outc.shape == (300, 516)
    np.savez_compressed(os.path.join(HERE, "vq_6d.npz"), out=outv, idx_body=ib.numpy(), idx_hand=ih.numpy(), pose_seed=621,
                        out_cont=outc[::3].copy(), out_cont_stride=3, out_cont_seam=outc[56:64].copy(), pose_seed_cont=623,
                        fp_vq=np.array(list(synth.fingerprint(vq6).values())))
    print("vq_6d", outv.shape, outc.shape, ib[0, :4].tolist())

    # ---- the demo flow: scripts/demo.py:158-246 (infer) with every wrapper built from one convert_to_6d config --------
    from scipy.io import wavfile

    class _RenderTool:                                  # visualise/rendering.py needs pyrender / ffmpeg: out of scope
        def __init__(self, *aa, **kk):
            self.calls = []

        def _render_sequences(self, wav, vertices_list, **kk):
            self.calls.append((wav, len(vertices_list), kk))

    for name, attrs in (("visualise", {}), ("visualise.rendering", {"RenderTool": _RenderTool})):
        m = types.ModuleType(name)
        m.__spec__ = importlib.machinery.ModuleSpec(name, None)
        m.__path__ = []
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
    import data_utils.utils as ref_du
    import scripts.demo as ref_demo
    import transformers
    from talkshow_b200.data_utils.utils import load_wav
    from talkshow_b200.nets.smplx_face import hf_layerdrop_uses_torch_rng   # reads transformers' source only
    from trainer.options import parse_args as ref_parse_args

    # file decoding as in make_golden.py's demo_flow: the 16 kHz int16 file's samples, unchanged
    ref_du.ta.load = lambda fn: load_wav(fn)
    ref_du.librosa.load = lambda fn, sr=16000: (load_wav(fn)[0].mean(0).numpy(), 16000)
    ref_demo.Wav2Vec2Processor.from_pretrained = staticmethod(lambda name: object())
    sec, nsamp, spk, seed = DEMO_SECONDS, DEMO_SAMPLES, DEMO_SPEAKER, DEMO_SEED
    x = (synth.synth_wave(1, 16000 * sec, seed=DEMO_WAVE_SEED)[0].numpy() * 20000).astype(np.int16)
    wav = os.path.join(tmp, "clip six.wav")
    wavfile.write(wav, 16000, x)
    torch.save({"generator": bp6}, os.path.join(tmp, "body6.pth"))
    torch.save({"generator": face6}, os.path.join(tmp, "face6.pth"))

    def demo_args(n, flags=()):
        return ref_parse_args().parse_args(["--config_file", "config/body_pixel.json", "--infer", "--audio_file", wav, "--id", str(spk),
                                            "--num_sample", str(n), "--body_model_path", os.path.join(tmp, "body6.pth"),
                                            "--face_model_path", os.path.join(tmp, "face6.pth")] + list(flags))

    dargs = demo_args(nsamp)
    dargs.gpu = "cpu"
    g_body = ref_demo.init_model(dargs.body_model_name, dargs.body_model_path, dargs, cfg)
    g_face = ref_demo.init_model(dargs.face_model_name, dargs.face_model_path, dargs, cfg)
    assert g_body.generator.dim == 512 and not g_face.generator.audio_middle.identity

    class _Smplx:                                       # smplx is not installed: get_vertices only needs .vertices / .body_pose
        def __call__(self, **kw):
            return types.SimpleNamespace(vertices=torch.zeros(1, 4, 3), body_pose=kw["body_pose"])

    rt = _RenderTool()
    out_dir = os.path.join(tmp, "visualise", "video", cfg.Log.name)
    os.makedirs(out_dir, exist_ok=True)
    os.chdir(tmp)                                       # infer() saves relative to the working directory
    torch.manual_seed(seed)
    ref_demo.infer(g_body, g_face, _Smplx(), rt, cfg, dargs)
    saved = np.load(os.path.join(out_dir, "clip six.npy"))
    frame = 16000 * sec * 30 // 16000
    assert saved.shape == (nsamp * frame, 265) and len(rt.calls) == 1 and rt.calls[0][1] == nsamp
    # the body codes of the samples, recomputed through the same modules with the same seed and draw order
    torch.manual_seed(seed)
    if hf_layerdrop_uses_torch_rng():
        for _ in range(len(g_face.generator.audio_encoder.encoder.layers)):
            torch.rand([])
    feats = ref_du.get_mfcc_ta(wav, sr=22000, fps=30, smlpx=True, type="mfcc")
    aud = torch.tensor(feats.transpose(1, 0)[None], dtype=torch.float32)
    audio = g_body.audioencoder(aud).unsqueeze(-1).repeat(1, 1, 1, 2)
    T = audio.shape[2]
    codes = [g_body.generator.generate(torch.tensor([spk]), shape=[T, 2], batch_size=1, aud_feat=audio) for _ in range(nsamp)]
    stand_args = demo_args(1, ["--stand"])
    stand_args.gpu = "cpu"
    torch.manual_seed(seed)
    ref_demo.infer(g_body, g_face, _Smplx(), rt, cfg, stand_args)
    saved_stand = np.load(os.path.join(out_dir, "clip six.npy"))
    assert saved_stand.shape == (frame, 265)
    torch.manual_seed(seed)
    n_first = draw_noise(2 * T, 1)                      # fingerprint of this host's CPU stream under the seed
    np.savez_compressed(os.path.join(HERE, "demo_flow_6d.npz"), saved=saved, saved_stand=saved_stand, codes=torch.cat(codes).numpy(),
                        seconds=sec, num_sample=nsamp, speaker=spk, seed=seed, wave_seed=DEMO_WAVE_SEED, log_name=str(cfg.Log.name),
                        frame=frame, noise_fp=noise_fp(n_first), hf_torch_layerdrop=int(hf_layerdrop_uses_torch_rng()),
                        transformers_version=transformers.__version__,
                        fp_face=np.array(list(synth.fingerprint(face6).values())),
                        fp_body=np.array(list(synth.fingerprint(bp6).values())))
    os.chdir(REF_DIR)
    print("demo_flow_6d", saved.shape, float(np.abs(saved).max()), torch.cat(codes)[:, :3].tolist())
    os.chdir(cwd)


if __name__ == "__main__":
    main()
