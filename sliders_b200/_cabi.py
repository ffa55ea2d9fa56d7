"""ctypes binding of libsb200.so (C ABI in include/sb200.h).

The product path has no CPU or PyTorch fallback: if the CUDA extension is missing or the device is not
sm_90 every entry point raises.  torch is used only for device memory, streams and torch.distributed.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libsb200.so")

EPI_BIAS, EPI_ROWBIAS, EPI_RESID, EPI_GEGLU, EPI_LORA = 1, 2, 4, 8, 16
CONV_PAD_BR = 32


class Sb200Error(RuntimeError):
    pass


class LoraArgs(C.Structure):
    """struct sb200_lora (include/sb200.h)."""

    _fields_ = [
        ("down", C.c_void_p),
        ("up", C.c_void_p),
        ("r", C.c_int),
        ("rt", C.c_int),
        ("group_n", C.c_int),
        ("scale", C.c_float),
        ("scale_dev", C.c_void_p),
        ("sample_scale", C.c_void_p),
        ("rows_per_sample", C.c_int),
    ]


_p, _i, _f, _i64, _d = C.c_void_p, C.c_int, C.c_float, C.c_int64, C.c_double
_LP = C.POINTER(LoraArgs)

# name -> argtypes (restype is int unless listed in _RESTYPE)
SIGNATURES = {
    "sb200_version": [],
    "sb200_last_error": [],
    "sb200_create": [_i, C.POINTER(_p)],
    "sb200_destroy": [_p],
    "sb200_gemm": [_p, _p, _p, _i, _p, _i, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p, _p, _i, _p, _i, _LP, _i],
    "sb200_conv3x3": [_p, _p, _p, _i, _p, _i, _i, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p, _i,
                      _LP, _i],
    "sb200_attention": [_p, _p, _p, _i, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _i, _f, _p],
    "sb200_attention_bwd": [_p, _p, _p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _p, _p, _p, _i, _p, _i, _p, _i,
                            _i, _i, _i, _i, _i, _f],
    "sb200_attention_bwd_ws": [_p, _p, _p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _p, _p, _p, _i, _p, _i, _p, _i,
                               _i, _i, _i, _i, _i, _f, _p, C.c_size_t],
    "sb200_gemm_splitk_f32": [_p, _p, _p, _i, _p, _i, _p, _i, _i, _i, _i, _p, C.c_size_t],
    "sb200_adam_f32": [_p, _p, _p, _i, C.c_longlong, _d, _d, _d, _d, _d, _i],
    "sb200_guided_step_loss": [_p, _p, _p, _p, _f, _p, _f, _f, _p, _i64, _i, _p, _p, _p, _p],
    "sb200_groupnorm_bwd": [_p, _p, _p, _i, _i, _p, _i, _i, _p, _p, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p, _p],
    "sb200_layernorm_bwd": [_p, _p, _p, _i, _p, _p, _i, _p, _i, _p, _i, _i, _i, _f],
    "sb200_geglu": [_p, _p, _p, _i, _p, _i, _i, _i],
    "sb200_geglu_bwd": [_p, _p, _p, _i, _p, _i, _p, _i, _i, _i],
    "sb200_add": [_p, _p, _p, _i, _p, _i, _p, _i, _p, _i, _i, _i],
    "sb200_upsample2x_bwd": [_p, _p, _p, _p, _i, _i, _i, _i],
    "sb200_zero_stuff": [_p, _p, _p, _p, _i, _i, _i, _i],
    "sb200_conv_out_bwd": [_p, _p, _p, _i, _p, _p, _i, _i, _i, _i],
    "sb200_colsum": [_p, _p, _p, _i, _p, _i, _i, _i],
    "sb200_lora_proj": [_p, _p, _p, _i, _p, _i, _p, _i, _i, _i, _i],
    "sb200_lora_wgrad": [_p, _p, _p, _i, _p, _p, _i, _i, _f, _i, _i, _i, _i, _p],
    "sb200_lora_rank_update": [_p, _p, _p, _i, _p, _p, _i, _f, _i, _i, _i],
    "sb200_lora_conv_proj": [_p, _p, _p, _i, _i, _p, _i, _i, _p, _p, _i, _i, _i, _i, _i],
    "sb200_lora_conv_wgrad": [_p, _p, _p, _i, _i, _p, _i, _i, _p, _p, _f, _i, _i, _i, _i, _i, _i, _p],
    "sb200_lora_conv_rank_update": [_p, _p, _p, _p, _p, _f, _i, _i, _i, _i, _i, _i],
    "sb200_adamw": [_p, _p, _p, _i, C.c_longlong, _d, _d, _d, _d, _d, _i],
    "sb200_groupnorm": [_p, _p, _p, _i, _i, _p, _i, _i, _p, _p, _p, _i, _i, _i, _i, _f, _i, _p],
    "sb200_layernorm": [_p, _p, _p, _i, _p, _p, _p, _i, _i, _i, _f],
    "sb200_small_linear": [_p, _p, _p, _i, _p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _LP, _p],
    "sb200_sinusoid": [_p, _p, _p, _i, _i, _p, _i],
    "sb200_conv_in": [_p, _p, _p, _i, _p, _p, _p, _i, _i, _i, _i],
    "sb200_conv_out": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i],
    "sb200_upsample2x": [_p, _p, _p, _p, _i, _i, _i, _i],
    "sb200_cfg_ddim": [_p, _p, _p, _i, _f, _p, _f, _f, _p, _p, _i, _i64],
    "sb200_cfg_step": [_p, _p, _p, _i, _f, _p, _f, _f, _p, _p, _i, _i64],
    "sb200_lora_compose": [_p, _p, _p, _p, _p, _i64, _i],
    "sb200_vae_conv_in_u8": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i],
    "sb200_vae_conv_out_u8": [_p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i],
    "sb200_vae_moments": [_p, _p, _p, _p, _p, _p, _p, _p, _f, _p, _i, _i, _i, _i],
    "sb200_vae_post_quant": [_p, _p, _p, _p, _p, _f, _p, _i, _i],
    "sb200_softmax_rows": [_p, _p, _p, _i, _p, _i, _i, _i, _f],
}
_RESTYPE = {"sb200_version": C.c_char_p, "sb200_last_error": C.c_char_p}

_lib: Optional[C.CDLL] = None


def lib_path() -> str:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load libsb200.so and declare every prototype.  Raises Sb200Error if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise Sb200Error(
            f"{_LIB_PATH} not found: build it with `make` (or __graft_entry__.build()). "
            "sliders_b200 has no CPU / PyTorch fallback for the UNet denoise path."
        )
    lib = C.CDLL(_LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = _RESTYPE.get(name, C.c_int)
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().sb200_last_error().decode("utf-8", "replace")
        raise Sb200Error(f"libsb200 status {status}: {msg}")


_handles = {}


def handle(device_index: int) -> C.c_void_p:
    """Per-device context (created on first use)."""
    h = _handles.get(device_index)
    if h is None:
        lib = load()
        h = C.c_void_p()
        check(lib.sb200_create(int(device_index), C.byref(h)))
        _handles[device_index] = h
    return h
