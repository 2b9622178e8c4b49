"""Helpers of the fp16-compute parity tests (not a test module): fp16 rounding, the fp16 form of the GEMM parity bar and the
oracle's weight as the fp16 fused kernels read it."""
import numpy as np
import torch

import oracle_c as oc
from gpu_helpers import rel_err, state_to_numpy


def f16_round(a: np.ndarray) -> np.ndarray:
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def np32(t: torch.Tensor) -> np.ndarray:
    return t.detach().float().cpu().numpy()


def assert_close_f16(a: np.ndarray, ref: np.ndarray, tol: float = 1e-3, ulps: float = 1.0):
    """||a - ref||_F / ||ref||_F <= tol AND no element further than `ulps` fp16 ulps (2^-10 of the binade of the largest
    reference magnitude) from the fp16-rounded reference."""
    e = rel_err(a, ref)
    scale = max(float(np.abs(ref).max()), 1e-30)
    ulp = 2.0 ** (np.floor(np.log2(scale)) - 10)            # fp16: 11 significant bits
    u = float(np.abs(a.astype(np.float64) - ref.astype(np.float64)).max() / ulp)
    assert e <= tol and u <= ulps + 0.01, f"rel_F={e:.3e} (tol {tol}), max err = {u:.2f} fp16 ulp of max|ref|"


def oracle_w32(c_oracle, packed, qs) -> np.ndarray:
    """The unrounded fp32 weight LUT[j] * absmax of the C oracle (a nested absmax resolved by the oracle too)."""
    st = state_to_numpy(packed, qs)
    n = int(np.prod(st["shape"]))
    if st["nested"]:
        absmax = oc.nested_absmax(c_oracle, st["code256"], st["absmax_u8"], st["absmax2"], st["offset"])
    else:
        absmax = st["absmax"]
    return oc.dequantize_nf4_f32(c_oracle, st["packed"], absmax, n).reshape(st["shape"])


def oracle_w16(c_oracle, packed, qs) -> np.ndarray:
    """The oracle's fp32 weight rounded to fp16 by numpy (as fp32 values): what `dequantize_4bit(...).to(fp16)` returns."""
    return f16_round(oracle_w32(c_oracle, packed, qs))
