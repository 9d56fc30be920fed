"""ctypes binding of the C ABI declared in ``include/ctrl_adapter_b200.h``.

The shared library is built in-tree by ``build.py`` (``__graft_entry__.build()``).  There is no CPU
fallback: if the library is missing, or a CUDA launch fails, the error is raised to the caller.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctrl_adapter_b200.so")

CA_MAX_TAPS = 9
ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2


class GemmDesc(C.Structure):
    _fields_ = [
        ("nsrc", C.c_int32),
        ("a", C.c_void_p * 2),
        ("a_channels", C.c_int32 * 2),
        ("a_c_off", C.c_int32 * 2),
        ("a_c_len", C.c_int32 * 2),
        ("a_dims", C.c_int64 * 4),
        ("a_strides", (C.c_int64 * 4) * 2),
        ("box", C.c_int32 * 4),
        ("ntaps", C.c_int32),
        ("tap_off", (C.c_int32 * 4) * CA_MAX_TAPS),
        ("tap_c_off", C.c_int32 * CA_MAX_TAPS),
        ("w", C.c_void_p),
        ("w_rows", C.c_int32),
        ("w_k_per_tap", C.c_int32),
        ("bias", C.c_void_p),
        ("out", C.c_void_p),
        ("out_fp32", C.c_int32),
        ("n_out", C.c_int32),
        ("out_dims", C.c_int32 * 4),
        ("out_strides", C.c_int64 * 4),
        ("act", C.c_int32),
        ("out_scale", C.c_float),
        ("rowvec", C.c_void_p),
        ("rowvec_strides", C.c_int64 * 4),
        ("residual", C.c_void_p),
        ("blend_src", C.c_void_p),
        ("res_strides", C.c_int64 * 4),
        ("blend_alpha", C.c_void_p),
        ("bn", C.c_int32),
    ]


class AttentionDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("batch", C.c_int32), ("heads", C.c_int32), ("lq", C.c_int32), ("lk", C.c_int32),
        ("head_dim_pad", C.c_int32),
        ("scale", C.c_float),
        ("q_row_stride", C.c_int64), ("q_batch_stride", C.c_int64),
        ("k_row_stride", C.c_int64), ("k_batch_stride", C.c_int64),
        ("v_row_stride", C.c_int64), ("v_batch_stride", C.c_int64),
        ("out_row_stride", C.c_int64), ("out_batch_stride", C.c_int64),
        ("kv_batch_div", C.c_int32),
    ]


# name -> argtypes (restype is int status unless listed in _RESTYPES)
_P, _I, _L, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
SIGNATURES = {
    "ca_abi_version": [],
    "ca_last_error": [],
    "ca_device_ok": [],
    "ca_gemm": [C.POINTER(GemmDesc), _P],
    "ca_attention": [C.POINTER(AttentionDesc), _P],
    "ca_groupnorm_stats": [_P, _I, _P, _I, _I, _L, _I, _P, _P],
    "ca_groupnorm_apply": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _F, _P, _P, _P, _I, _I, _P, _P],
    "ca_layernorm": [_P, _L, _I, _F, _P, _P, _P, _L, _P, _P, _P],
    "ca_timestep_embedding": [_P, _I, _I, _I, _F, _I, _P, _P],
    "ca_silu": [_P, _L, _P, _P],
    "ca_add": [_P, _P, _L, _P, _P],
    "ca_nchw_to_nhwc": [_P, _I, _I, _I, _L, _I, _P, _P],
    "ca_nhwc_to_nchw": [_P, _I, _I, _I, _L, _P, _I, _P],
    "ca_avgpool": [_P, _I, _I, _I, _I, _I, _I, _P, _P],
    "ca_upsample2x": [_P, _I, _I, _I, _I, _P, _P],
    "ca_router_weights": [_P, _P, _I, _I, _P, _P],
    "ca_router_merge": [_P, _P, _I, _L, _P, _P],
    "ca_softmax_rows": [_P, _L, _L, _P, _P],
    "ca_frame_conv_small": [_P, _I, _I, _L, _I, _I, _I, _P, _P, _P, _P],
    "ca_cfg_euler": [_P, _P, _P, _L, _F, _P, _I, _P, _P, _P],
    "ca_cfg_euler_v": [_P, _P, _P, _L, _P, _I, _L, _P, _I, _P, _P, _P],
    "ca_cfg_ddim": [_P, _P, _P, _L, _F, _P, _I, _I, _P, _P, _P],
    "ca_i2vgen_latent_encoder": [_P, _I, _I, _L, _I, _P, _P, _P],
    "ca_temporal_attention": [_P, _P, _P, _I, _I, _L, _I, _F, _L, _P, _P],
}
_RESTYPES = {"ca_last_error": C.c_char_p}

_lib = None


class CtrlAdapterB200Error(RuntimeError):
    pass


def load():
    """dlopen the in-tree library and bind every exported symbol.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CtrlAdapterB200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the hot path)")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, C.c_int)
    if lib.ca_abi_version() != 1:
        raise CtrlAdapterB200Error("ABI version mismatch between _lib.py and the shared library")
    _lib = lib
    return lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = load().ca_last_error().decode(errors="replace")
        exc = ValueError if status == 1 else CtrlAdapterB200Error
        raise exc(f"ctrl_adapter_b200 {what} failed (status {status}): {msg}")
