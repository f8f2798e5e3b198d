"""CPU (-m "not gpu"): the C-ABI library loads and exports every symbol include/talkshow_b200.h
declares (no compute calls), host-side mirrors of the reference interface behave like the
reference (config schema, flags, pose layout, sharding, noise contract, error conventions)."""
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

import talkshow_oracle as O
from conftest import GOLDEN, ROOT
from talkshow_b200 import _lib, synth


def test_header_symbols_exported():
    hdr = open(os.path.join(ROOT, "include", "talkshow_b200.h")).read()
    names = set(re.findall(r"\b(ts_[a-z0-9_]+)\s*\(", hdr))
    names -= {"ts_engine", "ts_tensor", "ts_status"}
    assert len(names) >= 24
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in sorted(names):
        assert hasattr(lib, n), "libtalkshow_b200.so does not export %s" % n
    # and the ctypes binding covers all of them
    assert names <= set(_lib.SYMBOLS), names - set(_lib.SYMBOLS)


def test_error_convention_without_gpu():
    L = _lib.lib()
    h = ctypes.c_void_p()
    if torch.cuda.is_available():
        pytest.skip("checks the no-device error path")
    rc = L.ts_engine_create(ctypes.byref(h), 0)
    assert rc != 0 and not h.value
    assert len(L.ts_last_error(None)) > 0
    assert L.ts_latent_rows(300) == 75 and L.ts_latent_rows(120) == 30 and L.ts_latent_rows(88) == 22


def test_host_only_engine_rejects_execution_and_bad_checkpoints():
    from talkshow_b200.engine import Engine

    e = Engine(-148)
    sd = synth.pixelcnn_state(0)
    bad = dict(sd)
    bad.pop("layers.3.horiz_resid.bias")
    with pytest.raises(RuntimeError, match="horiz_resid.bias"):
        e.load_pixelcnn(bad)
    bad = dict(sd)
    bad["fusion_v.weight"] = torch.zeros(256, 256, 1, 1)
    with pytest.raises(RuntimeError, match="fusion_v.weight"):
        e.load_pixelcnn(bad)
    with pytest.raises(RuntimeError, match="weight_norm"):
        e.load_face({})
    with pytest.raises(RuntimeError, match="embedding.weight"):
        e.load_pixelcnn(synth.body_pixel_checkpoint(0)["audioencoder"])          # the wrong module's dict
    e.load_pixelcnn(sd)
    assert e.pixelcnn_row_bytes == 89774080
    assert e.pixelcnn_staged_row_bytes > e.pixelcnn_row_bytes
    import ctypes as C
    ns, nc = C.c_int(0), C.c_int(0)
    assert e.L.ts_pixelcnn_plan_shape(e.h, C.byref(ns), C.byref(nc)) == 0 and (ns.value, nc.value) == (52, 148)
    with pytest.raises(RuntimeError, match="host-only"):
        e.pixelcnn_trace(0)
    # every executing entry point refuses a planning engine before it touches a pointer (no device copies of the weights exist)
    L, h, n = e.L, e.h, None
    for name, args in (("ts_audio_encode", (h, n, n, 1, 8, n)), ("ts_vq_decode", (h, 0, n, n, 1, 2, n)), ("ts_vq_encode", (h, 0, n, n, n, 1, 8, n)),
                       ("ts_face_forward", (h, n, n, n, 1, 16000, 30, n)), ("ts_body_generate", (h, n, n, n, n, n, 1, 8, n)),
                       ("ts_assemble_pose", (h, n, n, n, 1, 4, 4, 0, n)), ("ts_rot6d_to_axis_angle", (h, n, n, 4, n)),
                       ("ts_pixelcnn_generate", (h, n, n, n, n, n, 1, 2, n, 0, n)), ("ts_pixelcnn_timing", (h, 1)), ("ts_mfcc", (h, n, n, 1, 16000, 16000, n)),
                       ("ts_debug_conv1d", (h, n, n, n, n, n, n, n, n, n)), ("ts_debug_attention", (h, n, n, n, n, n, n)),
                       ("ts_debug_posconv", (h, 6, n, n, n, n, 1, 8, n)),
                       ("ts_debug_conv0_gn", (h, 6, n, n, n, n, n, n, n, 1, 400, n)), ("ts_debug_interp", (h, n, n, 1, 8, 5, 4, n)),
                       ("ts_debug_layernorm", (h, n, n, n, n, n, n, n, n, n, n)), ("ts_debug_vq_argmin", (h, n, 8, n, n, 4, n))):
        assert getattr(L, name)(*args) != 0 and b"host-only" in L.ts_last_error(h), name
    assert L.ts_set_vq_parallel(h, -1) != 0 and L.ts_set_vq_parallel(h, 16) == 0 and L.ts_set_pixelcnn_mode(h, 7) != 0
    with pytest.raises(ValueError):
        e.rot6d_to_axis_angle(torch.zeros(4, 5))
    e.close()


def test_wrappers_refuse_cpu_device():
    """No CPU fallback: the reference accepts args.gpu='cpu', the product must fail loudly."""
    from talkshow_b200.nets import s2g_body_pixel
    from talkshow_b200.trainer.config import load_JsonConfig

    cfg = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    with pytest.raises(RuntimeError, match="CUDA"):
        s2g_body_pixel(types.SimpleNamespace(gpu="cpu", infer=True), cfg)


def test_config_schema_matches_reference_fields():
    from talkshow_b200.trainer.config import load_JsonConfig

    for name in ("body_pixel", "body_vq", "face"):
        c = load_JsonConfig(os.path.join(ROOT, "config", name + ".json"))
        assert c.Data.pose.convert_to_6d is False and c.Data.pose.expression is True
        assert c.Data.pose.generate_length == 88 and c.Data.pose.normalization is False
        assert isinstance(c.Model.model_name, str) and isinstance(c.Log.name, str)
        assert c.Train.learning_rate.generator_learning_rate == 1e-4
    c = load_JsonConfig(os.path.join(ROOT, "config", "body_pixel.json"))
    assert c.Model.code_num == 2048 and c.Model.bh_model and c.Model.composition and c.Model.vq_path


def test_cli_flags():
    """parse_args() returns the PARSER like the reference (scripts/demo.py:251-252), and parses to the same namespace
    as the reference's parser — defaults and a demo command line, fixture written by make_golden.py --only options."""
    import argparse
    import json

    from talkshow_b200.trainer.options import parse_args

    gold = json.load(open(os.path.join(GOLDEN, "options.json")))
    parser = parse_args()
    assert isinstance(parser, argparse.ArgumentParser)
    assert vars(parser.parse_args([])) == gold["defaults"]
    assert vars(parse_args().parse_args(gold["demo_cmd"])) == gold["demo"]
    a = parse_args().parse_args(["--infer", "--audio_file", "x.wav", "--id", "2", "--num_sample", "12"])
    assert a.infer and a.id == 2 and a.num_sample == 12 and a.gpu == 0 and a.body_model_name == "s2g_body_pixel"


def test_pose_layout_helpers():
    from talkshow_b200.data_utils.lower_body import c_index_3d, part2full

    assert len(c_index_3d) == 129 and list(c_index_3d) == O.C_INDEX_3D
    x = torch.arange(3 * 232, dtype=torch.float32).view(3, 232)
    assert torch.equal(part2full(x), O.part2full(x))
    assert torch.equal(part2full(x, stand=True), O.part2full(x, stand=True))
    assert part2full(x).shape == (3, 265)


def test_pose_layout_matches_the_files_the_reference_ships():
    """demo/**/*.npy of the reference (written by its scripts/demo.py with the authors' checkpoints): (num_sample*F, 265) float32,
    the 33 columns part2full inserts are constant per file and equal this package's table in the sitting or the --stand variant; the
    --only_face file has the static 162-value body block.  Fixture: tests/golden/make_golden.py --only demo_npy_layout."""
    import json

    from talkshow_b200.data_utils.lower_body import part2full

    g = json.load(open(os.path.join(GOLDEN, "demo_npy_layout.json")))
    cols = g["lower_columns"]
    assert len(cols) == 33 and len(g["files"]) >= 8
    zero = torch.zeros(1, 232)
    sit = part2full(zero)[0, cols].tolist()
    stand = part2full(zero, stand=True)[0, cols].tolist()
    assert part2full(zero).shape == (1, 265) and sit != stand
    kinds = set()
    for name, f in g["files"].items():
        low = [np.float32(v) for v in f["lower"]]
        kind = "sit" if low == [np.float32(v) for v in sit] else "stand" if low == [np.float32(v) for v in stand] else None
        assert kind is not None, name
        kinds.add(kind)
        if f["only_face_static"] is not None:                       # scripts/demo.py:165-169,226-227
            static = torch.zeros(162)
            static[6:9] = torch.tensor([3.0747, -0.0158, -0.0152])
            assert [np.float32(v) for v in f["only_face_static"]] == [np.float32(v) for v in static.tolist()], name
            kinds.add("only_face")
    assert kinds == {"sit", "stand", "only_face"}


def test_lower_body_helpers_match_reference():
    """data_utils/lower_body.py of the reference, run on random inputs (tests/golden/make_golden.py --only lower_body): index tables and
    the four layout functions, bit for bit."""
    from talkshow_b200.data_utils import lower_body as lb

    g = np.load(os.path.join(GOLDEN, "lower_body.npz"))
    gen = torch.Generator().manual_seed(int(g["seed"]))
    pred, full, gt = torch.rand(6, 232, generator=gen), torch.rand(6, 265, generator=gen), torch.rand(4, 265, generator=gen)
    assert np.array_equal(lb.c_index_3d, g["c_index_3d"]) and np.array_equal(lb.c_index_6d, g["c_index_6d"])
    for name, got in (("part2full", lb.part2full(pred)), ("part2full_stand", lb.part2full(pred, True)), ("pred2poses", lb.pred2poses(pred, gt)),
                      ("poses2poses", lb.poses2poses(full, gt)), ("poses2pred", lb.poses2pred(full)), ("poses2pred_stand", lb.poses2pred(full, True))):
        assert np.array_equal(got.numpy(), g[name]), name


def test_shard_ranges_cover_batch():
    from talkshow_b200.pipeline import shard_range

    for B, G in ((12, 8), (64, 8), (12, 1), (5, 4), (64, 2)):
        r = [shard_range(B, k, G) for k in range(G)]
        assert r[0][0] == 0 and r[-1][1] == B
        assert all(r[i][1] == r[i + 1][0] for i in range(G - 1))
        assert max(hi - lo for lo, hi in r) - min(hi - lo for lo, hi in r) <= 1
    assert [hi - lo for lo, hi in (shard_range(12, k, 8) for k in range(8))] == [2, 2, 2, 2, 1, 1, 1, 1]


def test_noise_contract_matches_reference_multinomial():
    """draw_sampler_noise(per_step=True) consumes the generator exactly like the reference's
    probs.multinomial(1) calls: argmax(p/q) with our q == multinomial under the same seed."""
    from talkshow_b200.nets.base import draw_sampler_noise

    B, T = 3, 4
    probs = torch.softmax(torch.randn(2 * T, B, 2048, generator=torch.Generator().manual_seed(1)) * 3, -1)
    torch.manual_seed(77)
    ref = torch.stack([probs[s].multinomial(1).squeeze(-1) for s in range(2 * T)])
    torch.manual_seed(77)
    q = draw_sampler_noise(T, B, "cpu", per_step=True)
    assert torch.equal(torch.argmax(probs / q, -1), ref)


def test_front_end_matches_reference_functions(tmp_path):
    """get_mfcc_ta / get_mfcc_sepa (30 and 15 fps) on a stereo 44.1 kHz int16 file == the reference's functions on the same file
    (fixture: tests/golden/make_golden.py --only frontend; same torchaudio transforms, so the features are identical)."""
    from scipy.io import wavfile

    from talkshow_b200.data_utils.utils import get_mfcc_sepa, get_mfcc_ta

    g = np.load(os.path.join(GOLDEN, "frontend.npz"))
    x = (synth.synth_wave(2, int(g["sr"]) * int(g["seconds"]), seed=int(g["wave_seed"])).numpy().T * 20000).astype(np.int16)
    p = str(tmp_path / "stereo44k.wav")
    wavfile.write(p, int(g["sr"]), x)
    rows = []
    for fps in (30, 15):
        a = get_mfcc_ta(p, sr=22000, fps=fps, smlpx=True, type="mfcc", am=None)
        b, gap = get_mfcc_sepa(p, sr=22000, fps=fps)
        rows += [a.shape[0], b.shape[0]]
        assert gap == int(g["gap_%d" % fps])
        assert np.abs(a[::5] - g["ta_%d" % fps]).max() <= 1e-4 and np.abs(b[::5] - g["sepa_%d" % fps]).max() <= 1e-4
    assert [rows[0], rows[2], rows[1], rows[3]] == g["shapes"].tolist()


def test_mfcc_front_end_shapes(tmp_path):
    from scipy.io import wavfile

    from talkshow_b200.data_utils.utils import get_mfcc_ta

    sr = 16000
    x = (synth.synth_wave(1, sr * 4)[0].numpy() * 20000).astype(np.int16)
    p = str(tmp_path / "a.wav")
    wavfile.write(p, sr, np.stack([x, x], 1))          # stereo int16
    m = get_mfcc_ta(p, sr=22000, fps=30, smlpx=True, type="mfcc")
    assert m.shape == (120, 64) and np.isfinite(m).all()            # M = 4 s * 30 fps, SURVEY.md §8
    w = get_mfcc_ta(p, am=True, am_sr=16000, fps=30, encoder_choice="faceformer")
    assert w.shape == (sr * 4, 1)
    assert O.latent_rows(120) == 30
