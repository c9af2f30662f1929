"""ctypes binding of libd4d.so (C ABI in include/d4d.h).  There is NO fallback: if the CUDA library is
missing or fails, every call raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libd4d.so")

# every symbol include/d4d.h declares (tests check the library exports all of them)
EXPORTS = [
    "d4d_last_error", "d4d_version", "d4d_create", "d4d_destroy", "d4d_load_weight", "d4d_finalize_weights",
    "d4d_num_weights", "d4d_weight_key", "d4d_unet_forward", "d4d_profile_forward", "d4d_workspace_bytes", "d4d_forward_launches",
    "d4d_denoise_window", "d4d_assemble_input", "d4d_cfg_ddim_step", "d4d_op_gemm", "d4d_op_conv3x3",
    "d4d_op_attention", "d4d_op_groupnorm", "d4d_op_conv3x3_groupnorm", "d4d_op_conv_resample", "d4d_op_layernorm", "d4d_debug_tap", "d4d_exchange_alloc",
    "d4d_exchange_open", "d4d_unet_forward_sharded", "d4d_denoise_window_sharded",
]


class D4DConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int32), ("out_channels", C.c_int32), ("block_out_channels", C.c_int32 * 4),
        ("layers_per_block", C.c_int32), ("num_heads", C.c_int32 * 4), ("has_attn2", C.c_int32 * 4),
        ("use_linear_projection", C.c_int32), ("norm_num_groups", C.c_int32), ("norm_eps", C.c_float),
        ("flip_sin_to_cos", C.c_int32), ("freq_shift", C.c_float), ("num_3d_attn_blocks", C.c_int32),
        ("enable_tem_embeds", C.c_int32), ("enable_pose_encoder", C.c_int32), ("center_input_sample", C.c_int32),
    ]


class D4DSched(C.Structure):
    _fields_ = [
        ("timesteps_table", C.c_void_p), ("alphas_cumprod", C.c_void_p), ("n_steps", C.c_int32),
        ("num_train_timesteps", C.c_int32), ("final_alpha_cumprod", C.c_float), ("prediction_type", C.c_int32),
        ("clip_sample", C.c_int32), ("clip_sample_range", C.c_float), ("emulate_bf16", C.c_int32),
    ]


class D4DError(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Load libd4d.so (built by ``python -m diffuman4d_b200.build`` / ``__graft_entry__.build()``)."""
    global _lib
    if _lib is None:
        _lib = _load(LIB_PATH)
    return _lib


def _load(path: str) -> C.CDLL:
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: the CUDA extension is the product and there is no CPU fallback. "
            "Build it with `python -m diffuman4d_b200.build`.")
    l = C.CDLL(path)
    vp, i32, i64p, f32, f32p = C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.c_float, C.c_void_p
    l.d4d_last_error.restype = C.c_char_p
    l.d4d_last_error.argtypes = []
    l.d4d_version.restype = C.c_int
    l.d4d_create.argtypes = [C.POINTER(D4DConfig), i32, C.POINTER(vp)]
    l.d4d_destroy.argtypes = [vp]
    l.d4d_destroy.restype = None
    l.d4d_load_weight.argtypes = [vp, C.c_char_p, vp, i64p, i32, i32]
    l.d4d_finalize_weights.argtypes = [vp]
    l.d4d_num_weights.argtypes = [vp]
    l.d4d_weight_key.argtypes = [vp, i32]
    l.d4d_weight_key.restype = C.c_char_p
    l.d4d_unet_forward.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_int32), i32, i32, i32, i32, i32, vp, vp]
    l.d4d_profile_forward.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_int32), i32, i32, i32, i32, i32, vp, vp,
                                      C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_double)]
    l.d4d_workspace_bytes.argtypes = [vp, i32, i32, i32, i32, i32, C.POINTER(C.c_size_t)]
    l.d4d_forward_launches.argtypes = [vp, i32, i32, i32, i32, i32, C.POINTER(C.c_int)]
    l.d4d_denoise_window.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.POINTER(D4DSched), f32, i32, i32, i32, i32, i32, vp]
    l.d4d_assemble_input.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]
    l.d4d_cfg_ddim_step.argtypes = [vp, vp, vp, vp, vp, C.POINTER(D4DSched), f32, i32, i32, i32, i32, vp, vp]
    l.d4d_op_gemm.argtypes = [vp, i32, i32, vp, i32, i32, vp, i32, i32, f32p, vp, i32, i32, vp, i32, vp, i32, i32,
                              i32, f32, i32, vp]
    l.d4d_op_conv3x3.argtypes = [vp, i32, i32, i32, i32, vp, i32, f32p, vp, i32, vp, i32, vp, i32, vp]
    l.d4d_op_attention.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, f32, vp]
    l.d4d_op_groupnorm.argtypes = [vp, i32, vp, i32, i32, i32, i32, f32, f32p, f32p, i32, vp, vp]
    l.d4d_op_conv3x3_groupnorm.argtypes = [vp, i32, i32, i32, i32, vp, i32, f32p, vp, i32, f32, f32p, f32p, i32, vp, vp, vp]
    l.d4d_op_conv_resample.argtypes = [vp, i32, i32, i32, i32, vp, i32, f32p, i32, i32, i32, vp, vp]
    l.d4d_op_layernorm.argtypes = [vp, i32, i32, f32, f32p, f32p, vp, vp]
    l.d4d_debug_tap.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_int32), i32, i32, i32, i32, i32, i32, vp, C.c_char_p,
                                C.POINTER(C.c_int32), vp]
    l.d4d_exchange_alloc.argtypes = [vp, C.c_size_t, vp]
    l.d4d_exchange_open.argtypes = [vp, i32, i32, vp]
    l.d4d_unet_forward_sharded.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_int32), i32, i32, i32, i32, i32, i32, vp, vp]
    l.d4d_denoise_window_sharded.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.POINTER(D4DSched), f32, i32, i32, i32, i32,
                                             i32, i32, vp]
    for name in EXPORTS:
        fn = getattr(l, name)
        if fn.restype is C.c_int or name.startswith("d4d_op_") or name in (
                "d4d_create", "d4d_load_weight", "d4d_finalize_weights", "d4d_unet_forward", "d4d_denoise_window",
                "d4d_exchange_alloc", "d4d_exchange_open", "d4d_unet_forward_sharded", "d4d_denoise_window_sharded",
                "d4d_debug_tap"):
            fn.restype = C.c_int
    return l


def check(rc: int, what: str = ""):
    """Map C status codes to the reference's exception types (ValueError for argument errors)."""
    if rc == 0:
        return
    msg = lib().d4d_last_error().decode("utf-8", "replace")
    if rc == 1:
        raise ValueError(f"{what}: {msg}" if what else msg)
    raise D4DError(f"{what}: {msg} (status {rc})" if what else f"{msg} (status {rc})")
