"""ctypes binding of libtalkshow_b200.so (C ABI: include/talkshow_b200.h).

The library is the product's only compute path: if it cannot be loaded the import fails loudly —
there is no PyTorch / CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtalkshow_b200.so")

_lib = None


class ts_tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("dtype", C.c_int32), ("ndim", C.c_int32),
                ("shape", C.c_int64 * 6)]


class ts_sample_ctl(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float), ("min_p", C.c_float),
                ("logp_out", C.c_void_p), ("kept_out", C.c_void_p)]


SYMBOLS = {
    "ts_engine_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "ts_engine_destroy": (None, [C.c_void_p]),
    "ts_last_error": (C.c_char_p, [C.c_void_p]),
    "ts_engine_sm_count": (C.c_int, [C.c_void_p]),
    "ts_load_pixelcnn": (C.c_int, [C.c_void_p, C.POINTER(ts_tensor), C.c_int]),
    "ts_load_audioenc": (C.c_int, [C.c_void_p, C.POINTER(ts_tensor), C.c_int]),
    "ts_load_vq": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(ts_tensor), C.c_int]),
    "ts_load_face": (C.c_int, [C.c_void_p, C.POINTER(ts_tensor), C.c_int]),
    "ts_audio_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ts_latent_rows": (C.c_int, [C.c_int]),
    "ts_vq_dim": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_nccl_unique_id": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p]),
    "ts_nccl_init": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int]),
    "ts_allgather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "ts_load_smplx": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "ts_smplx_dims": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "ts_smplx_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "ts_pixelcnn_generate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "ts_pixelcnn_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p]),
    "ts_body_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                 C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p]),
    "ts_pixelcnn_sample_ctl": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_body_sample_ctl": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_int, C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_sampler_noise": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ts_pixelcnn_sample_seeded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_body_sample_seeded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_int, C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_pixelcnn_sample_anchored": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                              C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_body_sample_anchored": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_pixelcnn_sample_styled": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                            C.c_int, C.POINTER(ts_sample_ctl), C.c_void_p]),
    "ts_body_sample_styled": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(ts_sample_ctl),
                                        C.c_void_p]),
    "ts_pixelcnn_score_styled": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ts_pixelcnn_logits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                     C.c_void_p]),
    "ts_pixelcnn_score": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_int, C.c_void_p]),
    "ts_vq_decode": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ts_vq_encode": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ts_face_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_void_p]),
    "ts_body_generate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                   C.c_int, C.c_void_p]),
    "ts_assemble_pose": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                   C.c_int, C.c_void_p]),
    "ts_assemble_pose6d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p]),
    "ts_face_dim": (C.c_int, [C.c_void_p]),
    "ts_vq_score": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                              C.c_void_p]),
    "ts_face_score": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                C.c_int, C.c_int, C.c_void_p]),
    "ts_mfcc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ts_mfcc_frames": (C.c_int, [C.c_int, C.c_int]),
    "ts_launch_count": (C.c_int64, [C.c_void_p]),
    "ts_pixelcnn_row_bytes": (C.c_int64, [C.c_void_p]),
    "ts_pixelcnn_staged_row_bytes": (C.c_int64, [C.c_void_p]),
    "ts_pixelcnn_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_pixelcnn_last_ms": (C.c_double, [C.c_void_p]),
    "ts_debug_pixelcnn_plan": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p,
                                         C.POINTER(C.c_int64)]),
    "ts_set_pixelcnn_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_pixelcnn_trace": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_pixelcnn_plan_shape": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ts_pixelcnn_trace_read": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]),
    "ts_rot6d_to_axis_angle": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "ts_set_pixelcnn_fusion": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_set_pixelcnn_ctas": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_set_vq_parallel": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_set_tensor_cores": (C.c_int, [C.c_void_p, C.c_int]),
    "ts_debug_conv1d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "ts_debug_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ts_debug_posconv": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                   C.c_void_p]),
    "ts_debug_conv0_gn": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ts_debug_interp": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ts_debug_layernorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ts_debug_vq_argmin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
}


def lib():
    """Load the shared library (raises if it was not built: run ``python -m talkshow_b200.build``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "talkshow_b200: %s is missing — build it with `python -m talkshow_b200.build` "
                "(there is no CPU/PyTorch fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)     # AttributeError if the library does not export the symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def pack_tensors(sd):
    """state dict (name -> torch CPU tensor) -> (ts_tensor array, keep-alive list)."""
    keep = []
    arr = (ts_tensor * len(sd))()
    for i, (k, v) in enumerate(sd.items()):
        t = v.detach().to("cpu")
        if t.is_floating_point():
            t = t.to(torch.float32).contiguous()
            dt = 0
        else:
            t = t.to(torch.int64).contiguous()
            dt = 1
        name = k.encode()
        keep.append((t, name))
        arr[i].name = name
        arr[i].data = t.data_ptr()
        arr[i].dtype = dt
        arr[i].ndim = t.dim()
        for d in range(t.dim()):
            arr[i].shape[d] = t.shape[d]
    return arr, keep


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def plan_to_numpy(handle):
    """Export the PixelCNN execution plan (tests interpret it on the CPU)."""
    L = lib()
    tl, bl = C.c_int64(0), C.c_int64(0)
    rc = L.ts_debug_pixelcnn_plan(handle, None, C.byref(tl), None, C.byref(bl))
    if rc:
        raise RuntimeError(L.ts_last_error(handle).decode())
    table = np.zeros(tl.value, dtype=np.int32)
    blob = np.zeros(bl.value, dtype=np.float32)
    rc = L.ts_debug_pixelcnn_plan(handle, table.ctypes.data_as(C.c_void_p), C.byref(tl),
                                  blob.ctypes.data_as(C.c_void_p), C.byref(bl))
    if rc:
        raise RuntimeError(L.ts_last_error(handle).decode())
    return table, blob
