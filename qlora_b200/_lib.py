"""ctypes binding of libqlora_b200.so — the C-ABI declared in include/qlora_b200.h.

Mirrors the role of bitsandbytes' `cextension.py` + `lib.c*` calls [upstream], but every entry
point returns a status code that is turned into a Python exception here (upstream exit(1)s).
There is NO CPU fallback: if the library is missing, every op raises.
"""
from __future__ import annotations

import ctypes as ct
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libqlora_b200.so")

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}

_lib = None
_load_error: str | None = None

_vp, _i64, _i32 = ct.c_void_p, ct.c_int64, ct.c_int
_SIGS = {
    "qb200_version": ([], _i32),
    "qb200_has_fused_gemm": ([], _i32),
    "qb200_last_error": ([], ct.c_char_p),
    "qb200_set_quant_math": ([_i32], _i32),
    "qb200_get_quant_math": ([], _i32),
    "qb200_quantize_nf4": ([_vp, _i32, _i64, _i32, _vp, _vp, _vp], _i32),
    "qb200_quantize_blockwise_8bit": ([_vp, _vp, _i64, _i32, _vp, _vp, _vp], _i32),
    "qb200_dequantize_blockwise_8bit": ([_vp, _vp, _vp, _i64, _i32, _vp, _vp], _i32),
    "qb200_dequantize_nf4": ([_vp, _vp, _i64, _i32, _vp, _i32, _vp], _i32),
    "qb200_dequantize_nf4_nested": ([_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _i32, _vp], _i32),
    "qb200_nf4_linear_fwd": ([_vp] * 9 + [_i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_bwd_dx": ([_vp] * 8 + [_i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_fwd_lora": ([_vp] * 10 + [_i64, _vp, _i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_bwd_dx_lora": ([_vp] * 9 + [_i64, _vp, _i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_workspace_size": ([_i64, _i64, _i64, _i32], _i64),
    "qb200_nf4_linear_scratch_size": ([_i32, _i64, _i64, _i64, _i32], _i64),
    "qb200_adamw32bit_step": ([_vp, _i32, _vp, _vp, _vp, _i64, ct.c_float, ct.c_float, ct.c_float, ct.c_float, ct.c_float, _i32,
                               ct.c_float, _vp], _i32),
    "qb200_adamw32bit_step_dev": ([_vp, _i32, _vp, _vp, _vp, _i64, ct.c_float, ct.c_float, ct.c_float, ct.c_float, ct.c_float, _vp, _vp,
                                   _vp], _i32),
    "qb200_lion32bit_step_dev": ([_vp, _i32, _vp, _vp, _i64] + [ct.c_float] * 4 + [_vp, _vp, _vp], _i32),
    "qb200_rmsprop32bit_step_dev": ([_vp, _i32, _vp, _vp, _i64] + [ct.c_float] * 4 + [_vp, _vp, _vp], _i32),
    "qb200_ademamix32bit_step_dev": ([_vp, _i32, _vp, _vp, _vp, _vp, _i64] + [ct.c_float] * 9 + [_vp, _vp, _vp], _i32),
    "qb200_managed_alloc": ([_i64, ct.POINTER(ct.c_void_p)], _i32),
    "qb200_managed_free": ([_vp], _i32),
    "qb200_prefetch": ([_vp, _i64, _i32, _vp], _i32),
    "qb200_nf4_linear_ex": ([_i32] + [_vp] * 10 + [_i64, _vp, _i64, _i64, _i64, _vp, _i64, _vp], _i32),
    "qb200_nf4_linear_group": ([_i32, _i32, _vp, _i64, _i64, _i64, _i64, _i32, _vp, _i64, _vp], _i32),
    "qb200_nf4_linear_group_scaled": ([_i32, _i32, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _vp, _i64, _vp], _i32),
    "qb200_lora_project": ([_vp, _i64, _vp, ct.c_float, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_group_typed": ([_i32, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _vp, _i64, _vp], _i32),
    "qb200_lora_project_typed": ([_i32, _vp, _i64, _vp, ct.c_float, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_group_ex": ([_i32, _i32, _i32, _i32, _vp, _i64, _i64, _i64, _i64, _i32, _vp, _i64, _vp], _i32),
    "qb200_nf4_linear_group_reuse": ([_i32, _i32, _i32, _i32, _vp, _i64, _i64, _i64, _i64, _i32, _vp, _i64, ct.POINTER(_i32), _vp],
                                     _i32),
    "qb200_lora_project_mixed": ([_i32, _vp, _i64, _vp, _i32, _vp, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_nf4_linear_group_mixed": ([_i32, _i32, _i32, _vp, _i32, _vp, _i64, _i64, _i64, _i64, _i32, _vp], _i32),
    "qb200_lora_segment_workspace_size": ([_i64, _i32], _i64),
    "qb200_lora_segment_table": ([_vp, _i64, _i32, _vp, _i64, _vp], _i32),
    "qb200_lora_shrink_segmented": ([_i32, _i32, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_lora_expand_segmented": ([_i32, _i32, _vp, _vp, _i64, _vp, _i64, _i32, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_lora_grad_shrink_segmented": ([_i32, _i32, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_lora_grad_input_segmented": ([_i32, _i32, _i32, _vp, _vp, _i64, _vp, _i64, _i32, _vp, _i64, _i64, _i64, _i64, _vp], _i32),
    "qb200_lora_weight_grad_segmented": ([_i32, _i32, _i32, _vp, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _vp, _i64, _i64, _i64, _i64,
                                          _vp], _i32),
    "qb200_dora_stack_a": ([_i32, _i32, _vp, _vp, _vp, _i64, _vp, _i32, _i64, _i64, _vp], _i32),
    "qb200_dora_norm_segmented": ([_i32, _i32, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _i64, _i64, _vp],
                                  _i32),
    "qb200_dora_expand_segmented": ([_i32, _i32, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i32, _vp, _i64, _i64, _i64, _i64, _vp],
                                    _i32),
    "qb200_dora_grad_scale_segmented": ([_i32, _i32, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i32, _vp, _i64,
                                         _i64, _i64, _i64, _vp], _i32),
}


class Nf4Problem(ct.Structure):
    """`qb200_nf4_problem` of include/qlora_b200.h (one Linear4bit of a grouped launch)."""

    _fields_ = [("inp", _vp), ("ld_in", _i64), ("packed", _vp), ("absmax_u8", _vp), ("code256", _vp), ("absmax2", _vp),
                ("offset", _vp), ("absmax_f32", _vp), ("bias", _vp), ("U", _vp), ("ld_u", _i64), ("V", _vp), ("out", _vp),
                ("ld_out", _i64)]


class LoraAdapter(ct.Structure):
    """`qb200_lora_adapter` of include/qlora_b200.h (one entry of a mixed-adapter table)."""

    _fields_ = [("A", _vp), ("B", _vp), ("scale", ct.c_float), ("rank", ct.c_int32)]


# upstream-named aliases (bound here only so the export test can see them)
_COMPAT = [
    "cquantize_blockwise_fp32_nf4", "cquantize_blockwise_fp16_nf4", "cquantize_blockwise_bf16_nf4",
    "cdequantize_blockwise_fp32_nf4", "cdequantize_blockwise_fp16_nf4", "cdequantize_blockwise_bf16_nf4",
    "cquantize_blockwise_fp32", "cdequantize_blockwise_fp32",
]
EXPORTED_SYMBOLS = list(_SIGS) + _COMPAT


def load(required: bool = True):
    """Load (once) and return the ctypes library.  Raises if it cannot be loaded."""
    global _lib, _load_error
    if _lib is not None:
        return _lib
    if _load_error is None:
        try:
            lib = ct.CDLL(LIB_PATH)
            for name, (argtypes, restype) in _SIGS.items():
                fn = getattr(lib, name)
                fn.argtypes = argtypes
                fn.restype = restype
            for name in _COMPAT:
                getattr(lib, name)
            _lib = lib
            return _lib
        except (OSError, AttributeError) as e:  # missing file / missing symbol
            _load_error = f"{type(e).__name__}: {e}"
    if required:
        raise RuntimeError(
            f"qlora_b200: the CUDA extension {LIB_PATH} could not be loaded ({_load_error}). "
            "Build it with `python -m qlora_b200._build` (needs nvcc). There is no CPU fallback."
        )
    return None


def is_available() -> bool:
    return load(required=False) is not None


class Qb200Error(RuntimeError):
    pass


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().qb200_last_error().decode("utf-8", "replace")
        kind = "CUDA error" if rc > 0 else {-1: "invalid argument", -2: "unsupported shape", -3: "driver API"}.get(rc, "error")
        raise Qb200Error(f"{what} failed: {kind} {rc}: {msg}")


def ptr(t: torch.Tensor | None):
    return None if t is None else ct.c_void_p(t.data_ptr())


def stream_ptr(device: torch.device):
    return ct.c_void_p(torch.cuda.current_stream(device).cuda_stream)
