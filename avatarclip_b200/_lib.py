"""ctypes binding of libavc_b200.so (the C ABI declared in include/avc_b200.h).

There is NO fallback: if the CUDA library is missing, or a call returns an error code, this
module raises.  PyTorch is used by the callers only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libavc_b200.so")
# diagnostic builds (e.g. the NT stall probe of tools/nt_probe.py) live next to the product library
if os.environ.get("AVC_B200_LIB"):
    LIB_PATH = os.path.abspath(os.environ["AVC_B200_LIB"])

_ERR = {
    -1: "AVC_E_BADCFG (unsupported configuration)",
    -2: "AVC_E_NULL (required pointer is NULL)",
    -3: "AVC_E_SIZE (workspace too small / size mismatch)",
    -4: "AVC_E_ALIGN (pointer not 16-byte aligned)",
    -5: "AVC_E_NOSTASH",
}


class AvcError(RuntimeError):
    pass


class NeusCfg(C.Structure):
    _fields_ = [
        ("sdf_d_in", C.c_int32), ("sdf_d_out", C.c_int32), ("sdf_d_hidden", C.c_int32),
        ("sdf_n_layers", C.c_int32), ("sdf_skip_mask", C.c_uint32), ("sdf_multires", C.c_int32),
        ("sdf_scale", C.c_float),
        ("col_d_feature", C.c_int32), ("col_d_hidden", C.c_int32), ("col_n_layers", C.c_int32),
        ("n_samples", C.c_int32), ("n_importance", C.c_int32), ("up_sample_steps", C.c_int32),
        ("engine", C.c_int32), ("color_products", C.c_int32), ("wgrad_products", C.c_int32),
    ]


_OUT_FIELDS = ["color_fine", "extra_color_fine", "s_val", "cdf_fine", "weight_sum", "weight_max",
               "gradients", "weights", "mid_z_vals", "gradient_error", "inside_sphere", "z_vals"]
_COT_FIELDS = ["color_fine", "extra_color_fine", "s_val", "cdf_fine", "weight_sum", "weight_max",
               "gradients", "weights", "gradient_error"]


class NeusOutputs(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _OUT_FIELDS]


class NeusCotangents(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _COT_FIELDS]


_lib = None


def lib():
    """Load (once) and return the shared library; raise loudly when it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AvcError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  avatarclip_b200 has no CPU or PyTorch fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i64, i32, f32, sz = C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_size_t
    P = C.POINTER
    L.avc_abi_version.restype = C.c_int
    L.avc_build_arch.restype = C.c_char_p
    L.avc_neus_param_count.argtypes = [P(NeusCfg), P(i64)]
    L.avc_neus_param_offset.argtypes = [P(NeusCfg), C.c_int, C.c_int, C.c_int, P(i64), P(i64)]
    L.avc_neus_workspace_bytes.argtypes = [P(NeusCfg), i64, P(sz)]
    L.avc_neus_render_fwd.argtypes = [P(NeusCfg), vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, f32, i64,
                                      P(NeusOutputs), vp, sz, i64, vp]
    L.avc_neus_render_bwd.argtypes = [P(NeusCfg), vp, vp, vp, vp, C.c_int, f32, i64, P(NeusOutputs),
                                      P(NeusCotangents), vp, vp, sz, i64, i32, vp]
    L.avc_neus_sdf_query.argtypes = [P(NeusCfg), vp, vp, i64, vp, vp, sz, vp]
    L.avc_neus_sdf_eval.argtypes = [P(NeusCfg), vp, vp, i64, vp, vp, vp, sz, vp]
    L.avc_neus_sdf_eval.restype = C.c_int
    L.avc_march_count.argtypes = [vp, i32, i32, i32, f32, vp, vp]
    L.avc_march_emit.argtypes = [vp, i32, i32, i32, f32, vp, vp, vp, vp]
    L.avc_march_count.restype = L.avc_march_emit.restype = C.c_int
    L.avc_adam_step.argtypes = [vp, vp, vp, vp, i64, f32, f32, f32, f32, i64, f32, vp]
    L.avc_adam_step_dev.argtypes = [vp, vp, vp, vp, i64, vp, f32, f32, f32, f32, vp]
    L.avc_adam_step_dev.restype = C.c_int
    for name in ("avc_neus_param_count", "avc_neus_param_offset", "avc_neus_workspace_bytes",
                 "avc_neus_render_fwd", "avc_neus_render_bwd", "avc_neus_sdf_query", "avc_adam_step"):
        getattr(L, name).restype = C.c_int
    _lib = L
    return L


def check(rc: int, what: str):
    if rc == 0:
        return
    if rc < 0:
        raise AvcError(f"{what}: {_ERR.get(rc, rc)}")
    raise AvcError(f"{what}: CUDA error {rc}")


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
