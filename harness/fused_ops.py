"""ctypes binding + autograd wrappers of harness/csrc/fused_ops.cu (caller-side fusions for the bench harness;
not part of the qlora_b200 product).  `available()` is False when the library was not built — the harness then uses
the plain torch formulations."""
from __future__ import annotations

import ctypes as ct
import os
import shutil
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libharness_ops.so")
_SRC = os.path.join(_HERE, "csrc", "fused_ops.cu")
_lib = None


def build(force: bool = False) -> str:
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= os.path.getmtime(_SRC):
        return LIB_PATH
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-shared", "-o", LIB_PATH + ".tmp", _SRC, "-cudart", "static"], check=True)
    os.replace(LIB_PATH + ".tmp", LIB_PATH)
    return LIB_PATH


def _load():
    global _lib
    if _lib is None and os.path.exists(LIB_PATH):
        lib = ct.CDLL(LIB_PATH)
        vp, i64, i32 = ct.c_void_p, ct.c_int64, ct.c_int
        lib.hops_rope_qk.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i32, i32, i32, i32, ct.c_float, vp]
        lib.hops_swiglu_fwd.argtypes = [vp, vp, vp, i64, vp]
        lib.hops_swiglu_bwd.argtypes = [vp, vp, vp, vp, vp, i64, vp]
        lib.hops_rmsnorm_fwd.argtypes = [vp, vp, vp, vp, i64, i32, ct.c_float, vp]
        lib.hops_rmsnorm_bwd.argtypes = [vp, vp, vp, vp, vp, i64, i32, vp]
        lib.hops_dropout.argtypes = [vp, vp, i64, ct.c_float, vp, ct.c_uint64, vp]
        lib.hops_add_rmsnorm_fwd.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32, ct.c_float, vp]
        lib.hops_add_rmsnorm_bwd.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32, vp]
        for f in (lib.hops_rope_qk, lib.hops_swiglu_fwd, lib.hops_swiglu_bwd, lib.hops_rmsnorm_fwd, lib.hops_rmsnorm_bwd, lib.hops_dropout,
                  lib.hops_add_rmsnorm_fwd, lib.hops_add_rmsnorm_bwd):
            f.restype = i32
        _lib = lib
    return _lib


def available() -> bool:
    return _load() is not None


def _p(t):
    return ct.c_void_p(t.data_ptr())


def _s(t):
    return ct.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _rope(q, k, cos, sin_signed, sign):
    b, s, hq, d = q.shape
    hk = k.shape[2]
    qo, ko = torch.empty_like(q), torch.empty_like(k)
    rc = _load().hops_rope_qk(_p(q), _p(k), _p(qo), _p(ko), _p(cos), _p(sin_signed), b * s * hq, b * s * hk, hq, hk, s, d, sign, _s(q))
    if rc:
        raise RuntimeError(f"hops_rope_qk failed ({rc})")
    return qo, ko


class RopeQK(torch.autograd.Function):
    """q, k: [b, s, h, d] contiguous bf16; cos, sin_signed: [s, 1, d] bf16 (harness.llama_qlora._rope_tables)."""

    @staticmethod
    def forward(ctx, q, k, cos, sin_signed):
        ctx.save_for_backward(cos, sin_signed)
        return _rope(q.contiguous(), k.contiguous(), cos, sin_signed, 1.0)

    @staticmethod
    def backward(ctx, gq, gk):
        cos, sin_signed = ctx.saved_tensors
        dq, dk = _rope(gq.contiguous(), gk.contiguous(), cos, sin_signed, -1.0)
        return dq, dk, None, None


class SwiGLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, g, u):
        g, u = g.contiguous(), u.contiguous()
        out = torch.empty_like(g)
        rc = _load().hops_swiglu_fwd(_p(g), _p(u), _p(out), g.numel(), _s(g))
        if rc:
            raise RuntimeError(f"hops_swiglu_fwd failed ({rc})")
        ctx.save_for_backward(g, u)
        return out

    @staticmethod
    def backward(ctx, dy):
        g, u = ctx.saved_tensors
        dy = dy.contiguous()
        dg, du = torch.empty_like(g), torch.empty_like(u)
        rc = _load().hops_swiglu_bwd(_p(g), _p(u), _p(dy), _p(dg), _p(du), g.numel(), _s(g))
        if rc:
            raise RuntimeError(f"hops_swiglu_bwd failed ({rc})")
        return dg, du


class RMSNorm(torch.autograd.Function):
    """bf16 x [.., d], frozen fp32 weight [d]; fp32 statistics; no weight gradient (the norms are frozen in QLoRA)."""

    @staticmethod
    def forward(ctx, x, w, eps):
        x = x.contiguous()
        rows, d = x.numel() // x.shape[-1], x.shape[-1]
        y = torch.empty_like(x)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        rc = _load().hops_rmsnorm_fwd(_p(x), _p(w), _p(y), _p(rstd), rows, d, float(eps), _s(x))
        if rc:
            raise RuntimeError(f"hops_rmsnorm_fwd failed ({rc})")
        ctx.save_for_backward(x, w, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, rstd = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        rows, d = x.numel() // x.shape[-1], x.shape[-1]
        rc = _load().hops_rmsnorm_bwd(_p(x), _p(w), _p(dy), _p(dx), _p(rstd), rows, d, _s(x))
        if rc:
            raise RuntimeError(f"hops_rmsnorm_bwd failed ({rc})")
        return dx, None, None


class SeededDropout(torch.autograd.Function):
    """Dropout whose mask is a pure function of (device seed tensor, call-site salt, element index): identical in the
    forward, the checkpoint recompute and the backward; a new mask every step once the caller bumps the seed tensor
    (inside the captured step graph).  bf16, numel % 8 == 0."""

    @staticmethod
    def forward(ctx, x, p, seed, salt):
        x = x.contiguous()
        out = torch.empty_like(x)
        rc = _load().hops_dropout(_p(x), _p(out), x.numel(), float(p), _p(seed), int(salt), _s(x))
        if rc:
            raise RuntimeError(f"hops_dropout failed ({rc})")
        ctx.p, ctx.seed, ctx.salt = p, seed, salt
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        out = torch.empty_like(g)
        rc = _load().hops_dropout(_p(g), _p(out), g.numel(), float(ctx.p), _p(ctx.seed), int(ctx.salt), _s(g))
        if rc:
            raise RuntimeError(f"hops_dropout failed ({rc})")
        return out, None, None, None


def seeded_dropout(x, p, seed, salt):
    return SeededDropout.apply(x, p, seed, salt)


class AddRMSNorm(torch.autograd.Function):
    """(x + delta, rmsnorm(x + delta)) in one kernel; backward folds the residual-path gradient into the norm's backward:
    d(x) = d(delta) = g_sum + d(rmsnorm)/d(sum).  bf16, frozen fp32 weight, last dim <= 8192."""

    @staticmethod
    def forward(ctx, x, delta, w, eps):
        x, delta = x.contiguous(), delta.contiguous()
        rows, d = x.numel() // x.shape[-1], x.shape[-1]
        s = torch.empty_like(x)
        y = torch.empty_like(x)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        rc = _load().hops_add_rmsnorm_fwd(_p(x), _p(delta), _p(w), _p(s), _p(y), _p(rstd), rows, d, float(eps), _s(x))
        if rc:
            raise RuntimeError(f"hops_add_rmsnorm_fwd failed ({rc})")
        ctx.save_for_backward(s, w, rstd)
        return s, y

    @staticmethod
    def backward(ctx, g_sum, g_y):
        s, w, rstd = ctx.saved_tensors
        rows, d = s.numel() // s.shape[-1], s.shape[-1]
        if g_y is None:
            return g_sum, g_sum, None, None
        g_y = g_y.contiguous()
        gs = None if g_sum is None else g_sum.contiguous()
        dx = torch.empty_like(s)
        rc = _load().hops_add_rmsnorm_bwd(_p(s), _p(w), _p(g_y), None if gs is None else _p(gs), _p(dx), _p(rstd), rows, d, _s(s))
        if rc:
            raise RuntimeError(f"hops_add_rmsnorm_bwd failed ({rc})")
        return dx, dx, None, None


def add_rmsnorm(x, delta, w, eps):
    return AddRMSNorm.apply(x, delta, w, eps)


def rmsnorm(x, w, eps):
    return RMSNorm.apply(x, w, eps)


def rope_qk(q, k, cos, sin_signed):
    return RopeQK.apply(q, k, cos, sin_signed)


def swiglu(g, u):
    return SwiGLU.apply(g, u)
