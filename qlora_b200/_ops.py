"""The library's launches as torch custom ops (namespace `qlora_b200`), so that `torch.compile` traces through them.

Every device call of `functional` goes through one of these ops, in eager mode as under compile: the ctypes calls into
libqlora_b200.so live in the ops' implementations only.  Each op has a fake kernel that states its outputs' shapes, dtypes
and strides and runs the same argument checks as the launch, so a rejected call raises at trace time as it does eagerly.

A `QuantState` is not a valid op argument: the ops take its tensors (absmax, and for a nested state the second-level code,
absmax and offset) plus plain ints.  Outputs that a caller lends (`outs`, `out`, `absmax`) are declared in `mutates_args`.
The choice between the skinny, split-K, fused and scratch kernels (inside the C library) and between the library's LoRA
projection and cuBLAS (`lora_project`) is made inside the ops at every call, never by a Python branch on the token count,
so a graph traced with a symbolic token count serves every count (tests/test_gpu_compile.py checks two lengths, one
compilation).
"""
from __future__ import annotations

import ctypes as ct
from typing import Optional

import torch
from torch import Tensor

from . import _lib
from . import functional as F
from ._lib import DTYPE_CODE, check, ptr, stream_ptr

BLOCKSIZES = (4096, 2048, 1024, 512, 256, 128, 64)


def _device(*tensors: Optional[Tensor]) -> torch.device:
    """The one CUDA device of the tensors (None entries skipped)."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(
                "qlora_b200 ops run on CUDA tensors only (H100-native kernels, no CPU fallback); "
                f"got a tensor on {t.device}"
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"all tensors must be on the same GPU, found {dev} and {t.device}")
    if dev is None:
        raise RuntimeError("no tensors given")
    return dev


def _check_blocksize(blocksize: int) -> None:
    if blocksize not in BLOCKSIZES:
        raise ValueError(f"blocksize {blocksize} not in {BLOCKSIZES}")


def _check_state(absmax: Tensor, code2: Optional[Tensor], absmax2: Optional[Tensor], offset: Optional[Tensor]) -> None:
    """The state tensors as the kernels read them: uint8 codes with fp32 code / absmax2 / offset (nested), or fp32 absmax."""
    nested = code2 is not None
    assert (absmax2 is not None) == nested and (offset is not None) == nested, "nested state: code2, absmax2 and offset"
    if nested:
        assert absmax.dtype == torch.uint8 and code2.dtype == absmax2.dtype == offset.dtype == torch.float32, \
            "nested state: uint8 absmax, fp32 code2 / absmax2 / offset"
        assert code2.is_contiguous() and absmax2.is_contiguous(), "nested state tensors must be contiguous"
    else:
        assert absmax.dtype == torch.float32, "plain state: fp32 absmax"
    assert absmax.is_contiguous(), "absmax must be contiguous"


# ----------------------------------------------------------------------------------------------------------------------
# the grouped NF4 linear: forward and dX of 1..3 Linear4bit of one shape in one launch
# ----------------------------------------------------------------------------------------------------------------------

def _check_group(is_bwd, inputs, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, us, vs, outs,
                 out_dtype, row_scales, w_scratch):
    """Argument rules of `qb200_nf4_linear_group_reuse` / `_typed`, checked before any launch (and by the fake kernel).
    Returns (device, m, r, c_in, f_out, compute dtype, double-rounded weights, fused-kernel-only variant)."""
    n = len(packeds)
    assert 1 <= n <= 3 and len(inputs) == n and len(absmax) == n and len(code2) == n and len(absmax2) == n \
        and len(offset) == n, "1..3 problems, with one input and one state each"
    dev = _device(*inputs, *packeds, *absmax, *code2, *absmax2, *offset)
    for i in range(n):
        _check_state(absmax[i], code2[i], absmax2[i], offset[i])
    assert len({c is None for c in code2}) == 1, "grouped problems must share their quantization form"
    c_in, f_out = (n_out, k_in) if is_bwd else (k_in, n_out)
    m = inputs[0].shape[0]
    cdt = inputs[0].dtype
    assert cdt in (torch.bfloat16, torch.float16), f"inputs: bf16 or fp16, got {cdt}"
    for t in inputs:
        assert t.dim() == 2 and t.shape == (m, c_in) and t.dtype == cdt, f"input: expected {cdt} [{m}, {c_in}]"
    for p in packeds:
        assert p.dtype == torch.uint8 and p.numel() * 2 == n_out * k_in, "packed: uint8 holding N * K / 2 bytes"
    assert state_dtype in (torch.bfloat16, torch.float16, torch.float32), f"state dtype: 16/32-bit float, got {state_dtype}"
    twice = cdt == torch.bfloat16 and state_dtype == torch.float16
    out_ok = (cdt, torch.float32, torch.float16) if cdt == torch.bfloat16 else (cdt, torch.float32)
    assert out_dtype in out_ok, f"out_dtype: one of {out_ok}, got {out_dtype}"
    ex = twice or (cdt == torch.bfloat16 and out_dtype == torch.float16)
    assert not (ex and row_scales), "row scales need a bf16 or fp32 state and a bf16 or fp32 output"
    assert not biases or len(biases) == n, "one bias (or None) per problem"
    for b in biases:
        if b is not None:
            assert not is_bwd and b.numel() == n_out, "bias: N elements, forward only"
    assert len(us) == len(vs) and (not us or len(us) == n), "LoRA: one U and one V per problem, or none"
    r = us[0].shape[1] if us else 0
    for u, v in zip(us, vs):
        assert u.dim() == 2 and u.shape == (m, r) and u.dtype == cdt, f"U: expected {cdt} [{m}, {r}]"
        assert v.shape == ((r, k_in) if is_bwd else (n_out, r)) and v.dtype == cdt, "V: lora_A [r, K] (dX) or lora_B [N, r]"
    n_outs = 1 if is_bwd else n
    assert len(outs) == n_outs, f"outs: {n_outs} tensors"
    for o in outs:
        assert o.shape == (m, f_out) and o.stride(1) == 1 and o.dtype == out_dtype, f"out: {out_dtype} [{m}, {f_out}] rows"
    assert not row_scales or len(row_scales) == n, "one row scale (or None) per problem"
    for sc in row_scales:
        if sc is not None:
            assert sc.shape == (n_out,) and sc.dtype == torch.float32 and sc.device == dev, "row scale: fp32 [N] on the GPU"
    assert w_scratch is None or (not row_scales and w_scratch.dtype == torch.uint8 and w_scratch.device == dev)
    return dev, m, r, c_in, f_out, cdt, twice, ex


@torch.library.custom_op("qlora_b200::nf4_linear_group", mutates_args=("outs", "w_scratch"))
def nf4_linear_group(is_bwd: bool, inputs: list[Tensor], packeds: list[Tensor], absmax: list[Tensor],
                     code2: list[Optional[Tensor]], absmax2: list[Optional[Tensor]], offset: list[Optional[Tensor]],
                     n_out: int, k_in: int, state_dtype: torch.dtype, biases: list[Optional[Tensor]], us: list[Tensor],
                     vs: list[Tensor], outs: list[Tensor], out_dtype: torch.dtype, row_scales: list[Optional[Tensor]],
                     w_scratch: Optional[Tensor], return_scratch: bool) -> Tensor:
    """`functional.nf4_linear_group` on the state's tensors, writing its results into `outs` (one per problem forward, one
    for the dX).  Empty lists stand for None (`biases`, `us` / `vs`, `row_scales`: a non-empty `row_scales` selects the
    row-scaled launch even when every entry is None).  The outputs are lent rather than returned because torch cannot
    functionalize an op that both mutates a list and returns one.  A lent `w_scratch` is declared mutated too: a call off
    the scratch path uses it as its split-K workspace.

    Returns the scratch: with `return_scratch`, the workspace when the call left its bf16 weight copies there, or with
    `w_scratch` lent, a one-byte tensor when the GEMM read the lent copies; an empty tensor otherwise."""
    dev, m, r, c_in, f_out, cdt, twice, ex = _check_group(is_bwd, inputs, packeds, absmax, code2, absmax2, offset, n_out, k_in,
                                                          state_dtype, biases, us, vs, outs, out_dtype, row_scales, w_scratch)
    n = len(packeds)
    n_outs = 1 if is_bwd else n
    none = torch.empty(0, dtype=torch.uint8, device=dev)
    if m == 0:
        return none
    lib = _lib.load()
    keep = []  # tensors that must outlive the launch call
    probs = (_lib.Nf4Problem * n)()

    def _rowmajor(t, cols):
        if t.stride(1) != 1 or (t.stride(0) % 8) or t.stride(0) < cols or (t.data_ptr() % 16):
            t = t.contiguous()
            keep.append(t)
        return t

    for i in range(n):
        x = _rowmajor(inputs[i], c_in)
        packed = packeds[i]
        if not packed.is_contiguous():
            packed = packed.contiguous()
            keep.append(packed)
        pr = probs[i]
        pr.inp, pr.ld_in = x.data_ptr(), x.stride(0)
        pr.packed = packed.data_ptr()
        if code2[i] is not None:
            pr.absmax_u8, pr.code256, pr.absmax2, pr.offset = (absmax[i].data_ptr(), code2[i].data_ptr(), absmax2[i].data_ptr(),
                                                               offset[i].data_ptr())
        else:
            pr.absmax_f32 = absmax[i].data_ptr()
        b = biases[i] if biases else None
        if b is not None:
            b = b.to(cdt).contiguous()
            keep.append(b)
            pr.bias = b.data_ptr()
        if r:
            u = _rowmajor(us[i], r)
            v = vs[i]
            if not v.is_contiguous():
                v = v.contiguous()
                keep.append(v)
            pr.U, pr.ld_u, pr.V = u.data_ptr(), u.stride(0), v.data_ptr()
        if i < n_outs:
            o = outs[i]
            pr.out, pr.ld_out = o.data_ptr(), o.stride(0)
    scales = None
    if row_scales:
        scales = (ct.c_void_p * n)()
        for i, sc in enumerate(row_scales):
            if sc is None:
                continue
            if not sc.is_contiguous():
                sc = sc.contiguous()
                keep.append(sc)
            scales[i] = sc.data_ptr()
    ws_bytes = lib.qb200_nf4_linear_workspace_size(m, n_out, k_in, int(is_bwd)) if n == 1 else 0
    # training token counts under bf16 compute (bf16 or fp32 state, bf16 or fp32 output, no row scale): each W is dequantized
    # once into a bf16 scratch that a TMA-fed GEMM reads; one dequantize launch per problem precedes the GEMM, unless the
    # caller passes back the scratch of an earlier call (w_scratch)
    scratch = (lib.qb200_nf4_linear_scratch_size(n, m, n_out, k_in, int(is_bwd))
               if cdt == torch.bfloat16 and not ex and scales is None else 0)
    ws_bytes = max(ws_bytes, scratch)
    if w_scratch is not None:
        ws, ws_bytes = w_scratch, w_scratch.numel()
    else:
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes > 0 else None
    w_in_ws = ct.c_int(int(w_scratch is not None))
    what = (("nf4_linear_bwd_dx" if is_bwd else "nf4_linear_fwd") + ("_lora" if r else "") + (f"_x{n}" if n > 1 else "")
            + ("_scaled" if scales is not None else "") + ("_f16" if cdt == torch.float16 else "")
            + ("_sf16" if twice else "") + ("_of16" if ex and out_dtype == torch.float16 else ""))
    with torch.cuda.device(dev):
        ev = F._event_begin()
        if scales is None:
            rc = lib.qb200_nf4_linear_group_reuse(int(is_bwd), DTYPE_CODE[cdt], DTYPE_CODE[state_dtype], n, ct.addressof(probs), r,
                                                  m, n_out, k_in, DTYPE_CODE[out_dtype], ptr(ws), ws_bytes, ct.byref(w_in_ws),
                                                  stream_ptr(dev))
        else:
            rc = lib.qb200_nf4_linear_group_typed(int(is_bwd), DTYPE_CODE[cdt], n, ct.addressof(probs), ct.addressof(scales), r, m,
                                                  n_out, k_in, DTYPE_CODE[out_dtype], ptr(ws), ws_bytes, stream_ptr(dev))
        check(rc, what)
        F._event_end(what, m * n, n_out, k_in, ev)
    if w_in_ws.value and w_scratch is None:
        F.LAUNCH_COUNTER[0] += n   # the dequantize launches that wrote the scratch
    if return_scratch and w_in_ws.value:
        none = ws if w_scratch is None else torch.zeros(1, dtype=torch.uint8, device=dev)
    return none


@nf4_linear_group.register_fake
def _(is_bwd, inputs, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, us, vs, outs, out_dtype,
      row_scales, w_scratch, return_scratch):
    dev, m, r, c_in, f_out, cdt, twice, ex = _check_group(is_bwd, inputs, packeds, absmax, code2, absmax2, offset, n_out, k_in,
                                                          state_dtype, biases, us, vs, outs, out_dtype, row_scales, w_scratch)
    # whether the call leaves its weights in the workspace is decided by the library at run time
    size = torch.library.get_ctx().new_dynamic_size() if return_scratch else 0
    return inputs[0].new_empty((size,), dtype=torch.uint8)


# ----------------------------------------------------------------------------------------------------------------------
# the lora_A projection U = scale * x . A^T
# ----------------------------------------------------------------------------------------------------------------------

def _check_lora_project(x2d: Tensor, lora_a: Tensor) -> None:
    _device(x2d, lora_a)
    assert x2d.dim() == 2 and lora_a.dim() == 2 and lora_a.shape[1] == x2d.shape[1], "x2d [M, K] and lora_a [r, K]"
    assert lora_a.dtype == x2d.dtype, "x2d and lora_a of one dtype"


@torch.library.custom_op("qlora_b200::lora_project", mutates_args=())
def lora_project(x2d: Tensor, lora_a: Tensor, scale: float) -> Tensor:
    """U[M, r] = scale * x2d . lora_a^T.  A decode step (1..16 tokens, bf16 or fp16, K a multiple of 8, contiguous A) takes
    the library's one-launch projection (`qb200_lora_project` / `_typed`), which chains with the skinny kernel by
    programmatic dependent launch; every other call is one cuBLAS GEMM with the scale as its alpha.  The choice is made
    here, at run time, so that a graph traced with a symbolic token count serves both."""
    _check_lora_project(x2d, lora_a)
    dev = x2d.device
    m, k = x2d.shape
    r = lora_a.shape[0]
    if not (1 <= m <= F.LORA_PROJECT_MAX_TOKENS and k % 8 == 0 and x2d.dtype in (torch.bfloat16, torch.float16)
            and lora_a.is_contiguous()):
        u = torch.empty((m, r), dtype=x2d.dtype, device=dev)
        return torch.addmm(u, x2d, lora_a.t(), beta=0.0, alpha=scale, out=u)
    if x2d.stride(1) != 1 or x2d.stride(0) % 8 or x2d.stride(0) < k or x2d.data_ptr() % 16:
        x2d = x2d.contiguous()
    if not lora_a.is_contiguous() or lora_a.data_ptr() % 16:
        lora_a = lora_a.contiguous()
    u = torch.empty((m, r), dtype=x2d.dtype, device=dev)
    F.LAUNCH_COUNTER[0] += 1
    lib = _lib.load()
    with torch.cuda.device(dev):
        if x2d.dtype == torch.float16:
            rc = lib.qb200_lora_project_typed(DTYPE_CODE[torch.float16], ptr(x2d), x2d.stride(0), ptr(lora_a), float(scale), ptr(u),
                                              r, m, k, r, stream_ptr(dev))
        else:
            rc = lib.qb200_lora_project(ptr(x2d), x2d.stride(0), ptr(lora_a), float(scale), ptr(u), r, m, k, r, stream_ptr(dev))
        check(rc, "lora_project")
    return u


@lora_project.register_fake
def _(x2d, lora_a, scale):
    _check_lora_project(x2d, lora_a)
    return x2d.new_empty((x2d.shape[0], lora_a.shape[0]))


# ----------------------------------------------------------------------------------------------------------------------
# mixed-adapter batches: one LoRA adapter per token row, read from a device table
# ----------------------------------------------------------------------------------------------------------------------

def _check_mixed_rows(x2d: Tensor, table: Tensor, rows: Tensor, n_adapters: int, r: int) -> None:
    _device(x2d, table, rows)
    assert x2d.dim() == 2 and x2d.dtype in (torch.bfloat16, torch.float16), "x2d: bf16 or fp16 [M, K]"
    assert table.dtype == torch.uint8 and table.is_contiguous() and table.numel() == n_adapters * ct.sizeof(_lib.LoraAdapter), \
        "table: the contiguous bytes of n_adapters qb200_lora_adapter entries"
    assert rows.dtype == torch.int32 and rows.shape == (x2d.shape[0],) and rows.is_contiguous(), "rows: contiguous int32 [M]"
    assert 8 <= r <= F.LORA_MAX_RANK and r % 8 == 0, "R: a multiple of 8 in [8, 256]"


@torch.library.custom_op("qlora_b200::lora_project_mixed", mutates_args=())
def lora_project_mixed(x2d: Tensor, table: Tensor, rows: Tensor, n_adapters: int, r: int) -> Tensor:
    """U[M, r]: row t is scale_a . x2d[t] . A_a^T of its adapter a = rows[t] (`qb200_lora_project_mixed`), zero beyond that
    adapter's rank and for rows without an adapter (an index outside [0, n_adapters))."""
    _check_mixed_rows(x2d, table, rows, n_adapters, r)
    dev = x2d.device
    m, k = x2d.shape
    u = torch.empty((m, r), dtype=x2d.dtype, device=dev)
    if m == 0:
        return u
    if x2d.stride(1) != 1 or x2d.stride(0) % 8 or x2d.stride(0) < k or x2d.data_ptr() % 16:
        x2d = x2d.contiguous()
    F.LAUNCH_COUNTER[0] += 1
    with torch.cuda.device(dev):
        check(_lib.load().qb200_lora_project_mixed(DTYPE_CODE[x2d.dtype], ptr(x2d), x2d.stride(0), ptr(table), n_adapters, ptr(rows),
                                                   ptr(u), r, m, k, r, stream_ptr(dev)), "lora_project_mixed")
    return u


@lora_project_mixed.register_fake
def _(x2d, table, rows, n_adapters, r):
    _check_mixed_rows(x2d, table, rows, n_adapters, r)
    return x2d.new_empty((x2d.shape[0], r))


def _check_group_mixed(x2d, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, us, tables, rows,
                       n_adapters, outs):
    n = len(packeds)
    assert len(tables) == n and len(us) == n, "one adapter table and one U per problem"
    for t in tables:
        _check_mixed_rows(x2d, t, rows, n_adapters, us[0].shape[1])
    _check_group(False, [x2d] * n, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, [], [], outs,
                 outs[0].dtype if outs else x2d.dtype, [], None)
    r = us[0].shape[1]
    for u in us:
        assert u.shape == (x2d.shape[0], r) and u.dtype == x2d.dtype, f"U: {x2d.dtype} [M, {r}]"
    assert outs[0].dtype in (torch.bfloat16, torch.float16), "out: 16-bit"


@torch.library.custom_op("qlora_b200::nf4_linear_group_mixed", mutates_args=("outs",))
def nf4_linear_group_mixed(x2d: Tensor, packeds: list[Tensor], absmax: list[Tensor], code2: list[Optional[Tensor]],
                           absmax2: list[Optional[Tensor]], offset: list[Optional[Tensor]], n_out: int, k_in: int,
                           state_dtype: torch.dtype, biases: list[Optional[Tensor]], us: list[Tensor], tables: list[Tensor],
                           rows: Tensor, n_adapters: int, outs: list[Tensor]) -> None:
    """out_p = x2d . W_p^T (+bias_p) + U_p[t] . B_{p,a(t)}^T for 1..3 problems of one shape on one input, a decode step
    (`qb200_nf4_linear_group_mixed`): tables[p] is problem p's adapter table, U_p its `lora_project_mixed` output."""
    _check_group_mixed(x2d, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, us, tables, rows,
                       n_adapters, outs)
    n = len(packeds)
    m = x2d.shape[0]
    if m == 0:
        return
    dev = x2d.device
    keep = []
    if x2d.stride(1) != 1 or x2d.stride(0) % 8 or x2d.stride(0) < k_in or x2d.data_ptr() % 16:
        x2d = x2d.contiguous()
    probs = (_lib.Nf4Problem * n)()
    for i in range(n):
        packed = packeds[i] if packeds[i].is_contiguous() else packeds[i].contiguous()
        u = us[i] if us[i].is_contiguous() else us[i].contiguous()
        keep += [packed, u]
        pr = probs[i]
        pr.inp, pr.ld_in, pr.packed = x2d.data_ptr(), x2d.stride(0), packed.data_ptr()
        if code2[i] is not None:
            pr.absmax_u8, pr.code256, pr.absmax2, pr.offset = (absmax[i].data_ptr(), code2[i].data_ptr(), absmax2[i].data_ptr(),
                                                               offset[i].data_ptr())
        else:
            pr.absmax_f32 = absmax[i].data_ptr()
        b = biases[i] if biases else None
        if b is not None:
            b = b.to(x2d.dtype).contiguous()
            keep.append(b)
            pr.bias = b.data_ptr()
        pr.U, pr.ld_u, pr.V = u.data_ptr(), u.stride(0), tables[i].data_ptr()
        pr.out, pr.ld_out = outs[i].data_ptr(), outs[i].stride(0)
    what = "nf4_linear_fwd_mixed" + (f"_x{n}" if n > 1 else "") + ("_f16" if x2d.dtype == torch.float16 else "")
    with torch.cuda.device(dev):
        ev = F._event_begin()
        rc = _lib.load().qb200_nf4_linear_group_mixed(DTYPE_CODE[x2d.dtype], DTYPE_CODE[state_dtype], n, ct.addressof(probs),
                                                      n_adapters, ptr(rows), us[0].shape[1], m, n_out, k_in,
                                                      DTYPE_CODE[outs[0].dtype], stream_ptr(dev))
        check(rc, what)
        F._event_end(what, m * n, n_out, k_in, ev)


@nf4_linear_group_mixed.register_fake
def _(x2d, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, us, tables, rows, n_adapters, outs):
    _check_group_mixed(x2d, packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, biases, us, tables, rows,
                       n_adapters, outs)


# From this many (token rows x problems) on, U comes from the segmented tensor-core shrink, which reads each row of x once
# per 128 ranks but runs one CTA per 64-row tile and problem over the whole contraction; below it, from
# `qb200_lora_project_mixed`, which reads x once per rank but spreads a small batch over R x M / 8 CTAs.  On an H100 (r = 64,
# 1 to 16 adapters) the shrink was faster from 256 rows for q/k/v (3 problems, K = 4096) and from 1024 rows for down
# (1 problem, K = 11008), and slower at 512 rows for down.
SEGMENTED_SHRINK_MIN_WORK = 768


def _check_segmented(x2d: Tensor, tables: list[Tensor], rows: Tensor, n_adapters: int, r: int, outs: list[Tensor]) -> None:
    assert 1 <= len(tables) <= 3 and len(outs) == len(tables), "1..3 problems, one adapter table and one output each"
    for t in tables:
        _check_mixed_rows(x2d, t, rows, n_adapters, r)
    _device(x2d, *outs)
    m = x2d.shape[0]
    n_out = outs[0].shape[1] if outs else 0
    for o in outs:
        assert o.dim() == 2 and o.shape == (m, n_out) and o.dtype == x2d.dtype and o.is_contiguous(), \
            f"out: contiguous {x2d.dtype} [{m}, N]"
    assert n_out % 8 == 0, "N: a multiple of 8"


@torch.library.custom_op("qlora_b200::lora_segmented_add", mutates_args=("outs",))
def lora_segmented_add(x2d: Tensor, tables: list[Tensor], rows: Tensor, n_adapters: int, r: int, outs: list[Tensor]) -> None:
    """outs[p][t] = rn(outs[p][t] + U_p[t] . B_{p,a}^T) for every row t whose index a = rows[t] is in [0, n_adapters), with
    U_p[t] = rn(s_a . x2d[t] . A_{p,a}^T) of tables[p]; the other rows are not written.  Any token count, no host sync: the
    segment table (`qb200_lora_segment_table`), U (`qb200_lora_project_mixed` per problem when rows x
    problems is below SEGMENTED_SHRINK_MIN_WORK, else one `qb200_lora_shrink_segmented`) and one `qb200_lora_expand_segmented`
    for all problems.  The choice is made here at run time, so a graph traced with a symbolic token count serves both."""
    _check_segmented(x2d, tables, rows, n_adapters, r, outs)
    m = x2d.shape[0]
    if m == 0:
        return
    ws = torch.empty(segment_workspace_bytes(m, n_adapters), dtype=torch.uint8, device=x2d.device)
    _segmented_add([x2d], tables, rows, n_adapters, r, outs, [torch.empty((m, r), dtype=x2d.dtype, device=x2d.device) for _ in tables],
                   ws)


@lora_segmented_add.register_fake
def _(x2d, tables, rows, n_adapters, r, outs):
    _check_segmented(x2d, tables, rows, n_adapters, r, outs)


def segment_workspace_bytes(m, n_adapters: int):
    """`qb200_lora_segment_workspace_size(m, n_adapters)` (seg::layout in lora_segmented.cu), also for a symbolic m."""
    pad = lambda b: (b + 15) // 16 * 16  # noqa: E731
    return pad(4 * m) + pad(4 * (n_adapters + 2)) + 16 * ((m + 63) // 64 + n_adapters) + pad(8 * (n_adapters + 1))


def _rows_2d(t: Tensor) -> Tensor:
    """t as rows the segmented kernels read: unit stride, a row pitch of a multiple of 8 elements, 16-byte aligned."""
    if t.stride(1) != 1 or t.stride(0) % 8 or t.stride(0) < t.shape[1] or t.data_ptr() % 16:
        return t.contiguous()
    return t


def _segmented_add(xs, tables, rows, n_adapters, r, outs, us, ws, dora=None) -> None:
    """The segment table into `ws`, U_p into `us` and outs[p] += U_p . B^T: `lora_segmented_add` (one shared input in `xs`)
    and `lora_segmented_fwd` (one input per problem: each problem's U from its own input, one launch per problem).
    `dora` = (c [P, n, N], [Q_p] or []): the expand is `qb200_dora_expand_segmented` (`dora_segmented_fwd`)."""
    xs = [_rows_2d(x) for x in xs]
    m, k = xs[0].shape
    dev = xs[0].device
    n = len(tables)
    lib = _lib.load()
    ws_bytes = lib.qb200_lora_segment_workspace_size(m, n_adapters)
    assert ws_bytes > 0 and ws.numel() >= ws_bytes, "segmented LoRA: too many rows and adapters for one segment table"
    table_ptrs = (ct.c_void_p * n)(*[t.data_ptr() for t in tables])
    u_ptrs = (ct.c_void_p * n)(*[u.data_ptr() for u in us])
    out_ptrs = (ct.c_void_p * n)(*[o.data_ptr() for o in outs])
    dt = DTYPE_CODE[xs[0].dtype]
    shrink = m * n >= SEGMENTED_SHRINK_MIN_WORK
    F.LAUNCH_COUNTER[0] += 2 + (len(xs) if shrink else n)
    with torch.cuda.device(dev):
        s = stream_ptr(dev)
        check(lib.qb200_lora_segment_table(ptr(rows), m, n_adapters, ptr(ws), ws_bytes, s), "lora_segment_table")
        if shrink and len(xs) == 1:
            x2d = xs[0]
            check(lib.qb200_lora_shrink_segmented(dt, n, ptr(x2d), x2d.stride(0), table_ptrs, u_ptrs, r, n_adapters, ptr(ws), ws_bytes,
                                                  m, k, r, s), "lora_shrink_segmented")
        else:
            for i, (t, u) in enumerate(zip(tables, us)):
                x2d = xs[i % len(xs)]
                if shrink:
                    check(lib.qb200_lora_shrink_segmented(dt, 1, ptr(x2d), x2d.stride(0), (ct.c_void_p * 1)(t.data_ptr()),
                                                          (ct.c_void_p * 1)(u.data_ptr()), r, n_adapters, ptr(ws), ws_bytes, m, k,
                                                          r, s), "lora_shrink_segmented")
                else:
                    check(lib.qb200_lora_project_mixed(dt, ptr(x2d), x2d.stride(0), ptr(t), n_adapters, ptr(rows), ptr(u), r, m, k, r,
                                                       s), "lora_project_mixed")
        if dora is not None:
            cs, qs = dora
            check(lib.qb200_dora_expand_segmented(dt, n, int(bool(qs)), table_ptrs, u_ptrs, r, _ptrs(cs.unbind(0)),
                                                  _ptrs(qs) if qs else None, out_ptrs, outs[0].stride(0), n_adapters, ptr(ws),
                                                  ws_bytes, m, outs[0].shape[1], r, s), "dora_expand_segmented")
            return
        check(lib.qb200_lora_expand_segmented(dt, n, table_ptrs, u_ptrs, r, out_ptrs, outs[0].stride(0), n_adapters, ptr(ws),
                                              ws_bytes, m, outs[0].shape[1], r, s), "lora_expand_segmented")


# ----------------------------------------------------------------------------------------------------------------------
# training several adapters in one batch: the segmented forward that keeps U and the segment table, and its backward
# ----------------------------------------------------------------------------------------------------------------------

def _check_segmented_fwd(xs, tables, rows, n_adapters, r, outs) -> None:
    assert len(xs) in (1, len(tables)), "one input shared by the problems, or one per problem"
    for x in xs:
        _check_segmented(x, tables, rows, n_adapters, r, outs)
        assert x.shape == xs[0].shape, "the problems' inputs share one shape"


@torch.library.custom_op("qlora_b200::lora_segmented_fwd", mutates_args=("outs",))
def lora_segmented_fwd(xs: list[Tensor], tables: list[Tensor], rows: Tensor, n_adapters: int, r: int,
                       outs: list[Tensor]) -> tuple[Tensor, Tensor]:
    """`lora_segmented_add` that returns what the backward reads: (U [P, M, r], the segment table's workspace).  With one
    input in `xs` it runs exactly `lora_segmented_add`'s launches; with one input per problem (the adapters' dropped inputs),
    U_p is computed from xs[p]."""
    _check_segmented_fwd(xs, tables, rows, n_adapters, r, outs)
    m = xs[0].shape[0]
    dev = xs[0].device
    us = torch.empty((len(tables), m, r), dtype=xs[0].dtype, device=dev)
    ws = torch.empty(segment_workspace_bytes(m, n_adapters), dtype=torch.uint8, device=dev)
    if m:
        _segmented_add(xs, tables, rows, n_adapters, r, outs, list(us.unbind(0)), ws)
    return us, ws


@lora_segmented_fwd.register_fake
def _(xs, tables, rows, n_adapters, r, outs):
    _check_segmented_fwd(xs, tables, rows, n_adapters, r, outs)
    m = xs[0].shape[0]
    return xs[0].new_empty((len(tables), m, r)), xs[0].new_empty((segment_workspace_bytes(m, n_adapters),), dtype=torch.uint8)


def _check_segmented_bwd(g2ds, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dx, split):
    n = len(tables)
    assert 1 <= n <= 3 and len(g2ds) == n and len(xls) in (1, n), "1..3 problems: one dY each, one adapter input or one each"
    _device(*g2ds, *tables, rank_offsets, us, *xls, ws, dx)
    m, n_out = g2ds[0].shape
    cdt = g2ds[0].dtype
    assert cdt in (torch.bfloat16, torch.float16), "dY: bf16 or fp16"
    for g in g2ds:
        assert g.shape == (m, n_out) and g.dtype == cdt, f"dY: {cdt} [{m}, {n_out}]"
    k = xls[0].shape[1]
    for x in xls:
        assert x.dim() == 2 and x.shape == (m, k) and x.dtype == cdt, f"adapter input: {cdt} [{m}, K]"
    for t in tables:
        assert t.dtype == torch.uint8 and t.is_contiguous() and t.numel() == n_adapters * ct.sizeof(_lib.LoraAdapter), \
            "table: the contiguous bytes of n_adapters qb200_lora_adapter entries"
    assert rank_offsets.dtype == torch.int64 and rank_offsets.shape == (n_adapters,) and rank_offsets.is_contiguous(), \
        "rank_offsets: contiguous int64 [n_adapters]"
    assert 8 <= r <= F.LORA_MAX_RANK and r % 8 == 0 and rank_total >= 8, "R: a multiple of 8 in [8, 256]; rank_total >= 8"
    assert us.shape == (n, m, r) and us.dtype == cdt and us.is_contiguous(), f"U: contiguous {cdt} [{n}, {m}, {r}]"
    assert ws.dtype == torch.uint8 and ws.dim() == 1, "ws: the forward's segment table"
    assert n_out % 8 == 0 and k % 8 == 0, "N and K: multiples of 8"
    assert dx is None or (not split and dx.shape == (m, k) and dx.dtype == cdt and dx.stride(1) == 1), \
        f"dx: {cdt} [{m}, {k}] rows (no dropout input only)"
    assert not split or len(xls) == n, "split: one adapter input per problem"
    return m, n_out, k, cdt


@torch.library.custom_op("qlora_b200::lora_segmented_bwd", mutates_args=("dx",))
def lora_segmented_bwd(g2ds: list[Tensor], tables: list[Tensor], rank_offsets: Tensor, rank_total: int, us: Tensor,
                       xls: list[Tensor], ws: Tensor, n_adapters: int, r: int, dx: Optional[Tensor],
                       split: bool) -> tuple[Tensor, Tensor, Tensor]:
    """The LoRA part of a segmented backward, over the forward's U and segment table `ws`:
    G_p = rn(s_a . dY_p . B_{p,a}) (`qb200_lora_grad_shrink_segmented`); then, without dropout, dx += sum_p G_p . A_{p,a} in
    place on the base dX launch's output (or nothing when `dx` is None), with dropout (`split`) dxl_p = rn(G_p . A_{p,a}); and
    the flat weight gradients: dA [P, rank_total . K] (adapter a's [r_a, K] at rank_offsets[a] . K) and dB
    [P, rank_total . N] ([N, r_a] at rank_offsets[a] . N) (`qb200_lora_weight_grad_segmented`).
    Returns (dxl [P, M, K] with `split`, else an empty tensor; dA; dB)."""
    m, n_out, k, cdt = _check_segmented_bwd(g2ds, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dx, split)
    n = len(tables)
    dev = g2ds[0].device
    dxl = torch.zeros((n, m, k) if split else (0,), dtype=cdt, device=dev)
    d_a = torch.empty((n, rank_total * k), dtype=cdt, device=dev)
    d_b = torch.empty((n, rank_total * n_out), dtype=cdt, device=dev)
    if m == 0:
        return dxl, d_a.zero_(), d_b.zero_()
    g2ds = [g.contiguous() for g in g2ds]
    xls = [x.contiguous() for x in xls] * (n // len(xls))
    gs = torch.empty((n, m, r), dtype=cdt, device=dev)
    lib = _lib.load()
    ws_bytes = ws.numel()
    assert ws_bytes >= lib.qb200_lora_segment_workspace_size(m, n_adapters), "ws: the forward's segment table for these rows"
    arr = lambda ts: (ct.c_void_p * n)(*[t.data_ptr() for t in ts])  # noqa: E731
    tables_p, gs_p = arr(tables), arr(gs.unbind(0))
    dt = DTYPE_CODE[cdt]
    F.LAUNCH_COUNTER[0] += 3 + int(split or dx is not None)
    with torch.cuda.device(dev):
        s = stream_ptr(dev)
        check(lib.qb200_lora_grad_shrink_segmented(dt, n, arr(g2ds), n_out, tables_p, gs_p, r, n_adapters, ptr(ws), ws_bytes, m, n_out,
                                                   r, s), "lora_grad_shrink_segmented")
        if split:
            check(lib.qb200_lora_grad_input_segmented(dt, n, 0, tables_p, gs_p, r, arr(dxl.unbind(0)), k, n_adapters, ptr(ws),
                                                      ws_bytes, m, k, r, s), "lora_grad_input_segmented")
        elif dx is not None:
            check(lib.qb200_lora_grad_input_segmented(dt, n, 1, tables_p, gs_p, r, arr([dx] * n), dx.stride(0), n_adapters, ptr(ws),
                                                      ws_bytes, m, k, r, s), "lora_grad_input_segmented")
        check(lib.qb200_lora_weight_grad_segmented(dt, n, 0, tables_p, ptr(rank_offsets), rank_total, gs_p, r, arr(xls), k,
                                                   arr(d_a.unbind(0)), n_adapters, ptr(ws), ws_bytes, m, k, r, s),
              "lora_weight_grad_segmented")
        check(lib.qb200_lora_weight_grad_segmented(dt, n, 1, tables_p, ptr(rank_offsets), rank_total, arr(us.unbind(0)), r,
                                                   arr(g2ds), n_out, arr(d_b.unbind(0)), n_adapters, ptr(ws), ws_bytes, m, n_out,
                                                   r, s), "lora_weight_grad_segmented")
    return dxl, d_a, d_b


@lora_segmented_bwd.register_fake
def _(g2ds, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dx, split):
    m, n_out, k, cdt = _check_segmented_bwd(g2ds, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dx, split)
    n = len(tables)
    g = g2ds[0]
    return (g.new_empty((n, m, k) if split else (0,)), g.new_empty((n, rank_total * k)), g.new_empty((n, rank_total * n_out)))


# ----------------------------------------------------------------------------------------------------------------------
# training several DoRA adapters in one batch (DESIGN.md §6e): the norms of every adapter, the scaled expand and the
# gradient scale
# ----------------------------------------------------------------------------------------------------------------------

def _ptrs(ts):
    return (ct.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _check_tables(tables, n_adapters):
    for t in tables:
        assert t.dtype == torch.uint8 and t.is_contiguous() and t.numel() == n_adapters * ct.sizeof(_lib.LoraAdapter), \
            "table: the contiguous bytes of n_adapters qb200_lora_adapter entries"


def _check_dora_norm(tables, mag_tables, stack_rows, rank_offsets, gram_offsets, rank_total, gram_total, packeds, n_out, k_in,
                     row_norm2s, cdt, n_adapters, r):
    n = len(tables)
    assert 1 <= n <= 3 and len(mag_tables) == n and len(row_norm2s) == n and len(packeds) == n, \
        "1..3 problems: one adapter table, magnitude table, base and row norm each"
    _device(*tables, *mag_tables, stack_rows, rank_offsets, gram_offsets, *row_norm2s, *packeds)
    _check_tables(tables, n_adapters)
    for t in mag_tables:
        assert t.dtype == torch.int64 and t.shape == (n_adapters,) and t.is_contiguous(), "magnitude table: int64 [n_adapters]"
    for t in row_norm2s:
        assert t.dtype == torch.float32 and t.shape == (n_out,) and t.is_contiguous(), "row norms: contiguous fp32 [N]"
    assert stack_rows.dtype == torch.int32 and stack_rows.shape == (rank_total,) and stack_rows.is_contiguous(), \
        "stack_rows: contiguous int32 [rank_total]"
    for t in (rank_offsets, gram_offsets):
        assert t.dtype == torch.int64 and t.shape == (n_adapters,) and t.is_contiguous(), "offsets: contiguous int64 [n_adapters]"
    assert cdt in (torch.bfloat16, torch.float16), "compute dtype: bf16 or fp16"
    assert 8 <= r <= F.LORA_MAX_RANK and r % 8 == 0 and rank_total >= 8 and gram_total >= 64, "R: a multiple of 8 in [8, 256]"
    assert n_out % 8 == 0 and k_in % 8 == 0, "N and K: multiples of 8"


@torch.library.custom_op("qlora_b200::dora_segmented_norm", mutates_args=())
def dora_segmented_norm(tables: list[Tensor], mag_tables: list[Tensor], stack_rows: Tensor, rank_offsets: Tensor,
                        gram_offsets: Tensor, rank_total: int, gram_total: int, packeds: list[Tensor], absmax: list[Tensor],
                        code2: list[Optional[Tensor]], absmax2: list[Optional[Tensor]], offset: list[Optional[Tensor]], n_out: int,
                        k_in: int, state_dtype: torch.dtype, row_norm2s: list[Tensor], cdt: torch.dtype, n_adapters: int,
                        r: int) -> tuple[Tensor, Tensor]:
    """(c, n), fp32 [P, n_adapters, N]: DoRA's detached norm n_a = ||W_p + s_a B_a A_a||_row and c_a = m_a / n_a of every
    adapter of every problem, in a number of launches that does not depend on the adapters: `qb200_dora_stack_a` (each set's
    A matrices as rank_total rows), one grouped fused forward P_p = A_stack_p . W_p^T with an fp32 output, and
    `qb200_dora_norm_segmented` (the Gram matrices, then the per-row expansion of DESIGN.md §6b)."""
    _check_dora_norm(tables, mag_tables, stack_rows, rank_offsets, gram_offsets, rank_total, gram_total, packeds, n_out, k_in,
                     row_norm2s, cdt, n_adapters, r)
    n = len(tables)
    dev = packeds[0].device
    a_st = torch.empty((n, rank_total, k_in), dtype=cdt, device=dev)
    ps = torch.empty((n, rank_total, n_out), dtype=torch.float32, device=dev)
    gram = torch.empty((n, gram_total), dtype=torch.float32, device=dev)
    cs = torch.empty((n, n_adapters, n_out), dtype=torch.float32, device=dev)
    nrms = torch.empty_like(cs)
    lib = _lib.load()
    dt = DTYPE_CODE[cdt]
    tables_p = _ptrs(tables)
    F.LAUNCH_COUNTER[0] += 3
    with torch.cuda.device(dev):
        check(lib.qb200_dora_stack_a(dt, n, tables_p, ptr(stack_rows), ptr(rank_offsets), rank_total, _ptrs(a_st.unbind(0)),
                                     n_adapters, k_in, r, stream_ptr(dev)), "dora_stack_a")
    nf4_linear_group(False, list(a_st.unbind(0)), packeds, absmax, code2, absmax2, offset, n_out, k_in, state_dtype, [], [], [],
                     list(ps.unbind(0)), torch.float32, [], None, False)
    with torch.cuda.device(dev):
        check(lib.qb200_dora_norm_segmented(dt, n, tables_p, _ptrs(mag_tables), ptr(rank_offsets), ptr(gram_offsets), rank_total,
                                            gram_total, _ptrs(ps.unbind(0)), _ptrs(row_norm2s), _ptrs(gram.unbind(0)),
                                            _ptrs(cs.unbind(0)), _ptrs(nrms.unbind(0)), n_adapters, n_out, k_in, r, stream_ptr(dev)),
              "dora_norm_segmented")
    return cs, nrms


@dora_segmented_norm.register_fake
def _(tables, mag_tables, stack_rows, rank_offsets, gram_offsets, rank_total, gram_total, packeds, absmax, code2, absmax2, offset,
      n_out, k_in, state_dtype, row_norm2s, cdt, n_adapters, r):
    _check_dora_norm(tables, mag_tables, stack_rows, rank_offsets, gram_offsets, rank_total, gram_total, packeds, n_out, k_in,
                     row_norm2s, cdt, n_adapters, r)
    cs = row_norm2s[0].new_empty((len(tables), n_adapters, n_out))
    return cs, torch.empty_like(cs)


def _check_dora_fwd(xs, tables, rows, n_adapters, r, cs, outs, qs):
    _check_segmented_fwd(xs, tables, rows, n_adapters, r, outs)
    n, m, n_out = len(tables), xs[0].shape[0], outs[0].shape[1]
    _device(cs, *qs)
    assert cs.dtype == torch.float32 and cs.shape == (n, n_adapters, n_out) and cs.is_contiguous(), "c: contiguous fp32 [P, n, N]"
    assert not qs or (len(qs) == n and len(xs) == n), "Q: one per problem, with one dropped input per problem"
    for q in qs:
        assert q.shape == (m, n_out) and q.dtype == xs[0].dtype and q.stride() == outs[0].stride(), "Q: of the outputs' layout"


@torch.library.custom_op("qlora_b200::dora_segmented_fwd", mutates_args=("outs", "qs"))
def dora_segmented_fwd(xs: list[Tensor], tables: list[Tensor], rows: Tensor, n_adapters: int, r: int, cs: Tensor,
                       outs: list[Tensor], qs: list[Tensor]) -> tuple[Tensor, Tensor]:
    """`lora_segmented_fwd` with DoRA's magnitude scale `cs` (fp32 [P, n, N], `dora_segmented_norm`) in the expand
    (`qb200_dora_expand_segmented`): without dropout (`qs` empty) outs[p][t] = rn(c_a . (outs[p][t] + U_p[t] . B_a^T)); with
    it outs[p][t] = rn(outs[p][t] + (c_a - 1) . Q_p[t] + c_a . U_p[t] . B_a^T), Q_p = rn(Q_p + U_p . B_a^T) in place, Q_p
    given as rn(xs[p] . W_p^T).  Returns (U [P, M, r], the segment table's workspace)."""
    _check_dora_fwd(xs, tables, rows, n_adapters, r, cs, outs, qs)
    m = xs[0].shape[0]
    dev = xs[0].device
    us = torch.empty((len(tables), m, r), dtype=xs[0].dtype, device=dev)
    ws = torch.empty(segment_workspace_bytes(m, n_adapters), dtype=torch.uint8, device=dev)
    if m:
        _segmented_add(xs, tables, rows, n_adapters, r, outs, list(us.unbind(0)), ws, dora=(cs, qs))
    return us, ws


@dora_segmented_fwd.register_fake
def _(xs, tables, rows, n_adapters, r, cs, outs, qs):
    _check_dora_fwd(xs, tables, rows, n_adapters, r, cs, outs, qs)
    m = xs[0].shape[0]
    return xs[0].new_empty((len(tables), m, r)), xs[0].new_empty((segment_workspace_bytes(m, n_adapters),), dtype=torch.uint8)


def _check_dora_scale(g2ds, tables, rank_offsets, rank_total, qs, cs, nrms, ws, n_adapters, r, split):
    n = len(tables)
    assert 1 <= n <= 3 and len(g2ds) == n and len(qs) == n, "1..3 problems: one dY and one Q (or y) each"
    _device(*g2ds, *tables, rank_offsets, *qs, cs, nrms, ws)
    _check_tables(tables, n_adapters)
    m, n_out = g2ds[0].shape
    cdt = g2ds[0].dtype
    assert cdt in (torch.bfloat16, torch.float16), "dY: bf16 or fp16"
    for t in (*g2ds, *qs):
        assert t.shape == (m, n_out) and t.dtype == cdt and t.is_contiguous(), f"dY, Q: contiguous {cdt} [{m}, {n_out}]"
    for t in (cs, nrms):
        assert t.dtype == torch.float32 and t.shape == (n, n_adapters, n_out) and t.is_contiguous(), "c, n: fp32 [P, n, N]"
    assert rank_offsets.dtype == torch.int64 and rank_offsets.shape == (n_adapters,), "rank_offsets: int64 [n_adapters]"
    assert 8 <= r <= F.LORA_MAX_RANK and r % 8 == 0 and rank_total >= 8 and n_out % 8 == 0, "R: a multiple of 8 in [8, 256]"
    assert ws.dtype == torch.uint8 and ws.dim() == 1, "ws: the forward's segment table"
    return m, n_out, cdt


@torch.library.custom_op("qlora_b200::dora_grad_scale", mutates_args=())
def dora_grad_scale(g2ds: list[Tensor], tables: list[Tensor], rank_offsets: Tensor, rank_total: int, qs: list[Tensor], cs: Tensor,
                    nrms: Tensor, ws: Tensor, n_adapters: int, r: int, split: bool) -> tuple[Tensor, Tensor, Tensor]:
    """`qb200_dora_grad_scale_segmented` over the forward's segment table: (dQ [P, M, N] = rn(dY . c_a), dD [P, M, N] =
    rn(dY . (c_a - 1)) with `split` (else an empty tensor), dm [P, n . N] = rn(sum_t dY . Q / n_a) of the compute dtype).
    `qs`: the expand's Q_p with `split`, else the forward's outputs y_p (Q = y / c)."""
    m, n_out, cdt = _check_dora_scale(g2ds, tables, rank_offsets, rank_total, qs, cs, nrms, ws, n_adapters, r, split)
    n = len(tables)
    dev = g2ds[0].device
    dq = torch.empty((n, m, n_out), dtype=cdt, device=dev)
    dd = torch.empty((n, m, n_out) if split else (0,), dtype=cdt, device=dev)
    dm = torch.empty((n, n_adapters * n_out), dtype=cdt, device=dev)
    if m == 0:
        return dq, dd, dm.zero_()
    lib = _lib.load()
    assert ws.numel() >= lib.qb200_lora_segment_workspace_size(m, n_adapters), "ws: the forward's segment table for these rows"
    F.LAUNCH_COUNTER[0] += 1
    with torch.cuda.device(dev):
        check(lib.qb200_dora_grad_scale_segmented(DTYPE_CODE[cdt], n, int(split), _ptrs(tables), ptr(rank_offsets), rank_total,
                                                  _ptrs(g2ds), _ptrs(qs), _ptrs(cs.unbind(0)), _ptrs(nrms.unbind(0)), n_out,
                                                  _ptrs(dq.unbind(0)), _ptrs(dd.unbind(0)) if split else None, _ptrs(dm.unbind(0)),
                                                  n_adapters, ptr(ws), ws.numel(), m, n_out, r, stream_ptr(dev)),
              "dora_grad_scale_segmented")
    return dq, dd, dm


@dora_grad_scale.register_fake
def _(g2ds, tables, rank_offsets, rank_total, qs, cs, nrms, ws, n_adapters, r, split):
    m, n_out, cdt = _check_dora_scale(g2ds, tables, rank_offsets, rank_total, qs, cs, nrms, ws, n_adapters, r, split)
    n, g = len(tables), g2ds[0]
    return g.new_empty((n, m, n_out)), g.new_empty((n, m, n_out) if split else (0,)), g.new_empty((n, n_adapters * n_out))


def _check_dora_bwd(dqs, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dxs):
    n = len(tables)
    m, k = xls[0].shape
    _check_segmented_bwd(dqs, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, None, len(xls) > 1)
    assert len(dxs) in (1, n) and (len(dxs) == 1) == (len(xls) == 1), "one dx (no dropout) or one dxd per problem"
    for d in dxs:
        assert d.shape == (m, k) and d.dtype == dqs[0].dtype and d.stride(1) == 1, f"dx: {dqs[0].dtype} [{m}, {k}] rows"
    return m, dqs[0].shape[1], k, dqs[0].dtype


@torch.library.custom_op("qlora_b200::dora_segmented_bwd", mutates_args=("dxs",))
def dora_segmented_bwd(dqs: list[Tensor], tables: list[Tensor], rank_offsets: Tensor, rank_total: int, us: Tensor,
                       xls: list[Tensor], ws: Tensor, n_adapters: int, r: int, dxs: list[Tensor]) -> tuple[Tensor, Tensor]:
    """The adapters' part of a segmented DoRA backward, over dQ_p = rn(dY_p . c): G_p = rn(s_a . dQ_p . B_{p,a}); the input
    term added in place to the base dX launches' outputs, dxs[0] += sum_p G_p . A_{p,a} (one shared input) or dxs[p] +=
    G_p . A_{p,a} (one dropped input per problem), one rounding each; and the flat dA [P, rank_total . K] = G^T . xl and
    dB [P, rank_total . N] = dQ^T . U, laid out as `lora_segmented_bwd`'s."""
    m, n_out, k, cdt = _check_dora_bwd(dqs, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dxs)
    n = len(tables)
    dev = dqs[0].device
    d_a = torch.empty((n, rank_total * k), dtype=cdt, device=dev)
    d_b = torch.empty((n, rank_total * n_out), dtype=cdt, device=dev)
    if m == 0:
        return d_a.zero_(), d_b.zero_()
    dqs = [g.contiguous() for g in dqs]
    xls = [x.contiguous() for x in xls] * (n // len(xls))
    gs = torch.empty((n, m, r), dtype=cdt, device=dev)
    lib = _lib.load()
    ws_bytes = ws.numel()
    assert ws_bytes >= lib.qb200_lora_segment_workspace_size(m, n_adapters), "ws: the forward's segment table for these rows"
    tables_p, gs_p = _ptrs(tables), _ptrs(gs.unbind(0))
    dt = DTYPE_CODE[cdt]
    F.LAUNCH_COUNTER[0] += 3 + len(dxs)
    with torch.cuda.device(dev):
        s = stream_ptr(dev)
        check(lib.qb200_lora_grad_shrink_segmented(dt, n, _ptrs(dqs), n_out, tables_p, gs_p, r, n_adapters, ptr(ws), ws_bytes, m,
                                                   n_out, r, s), "lora_grad_shrink_segmented")
        if len(dxs) == 1:
            check(lib.qb200_lora_grad_input_segmented(dt, n, 1, tables_p, gs_p, r, _ptrs(dxs * n), dxs[0].stride(0), n_adapters,
                                                      ptr(ws), ws_bytes, m, k, r, s), "lora_grad_input_segmented")
        else:
            for p in range(n):
                check(lib.qb200_lora_grad_input_segmented(dt, 1, 1, _ptrs(tables[p:p + 1]), _ptrs(gs[p:p + 1].unbind(0)), r,
                                                          _ptrs(dxs[p:p + 1]), dxs[p].stride(0), n_adapters, ptr(ws), ws_bytes, m,
                                                          k, r, s), "lora_grad_input_segmented")
        check(lib.qb200_lora_weight_grad_segmented(dt, n, 0, tables_p, ptr(rank_offsets), rank_total, gs_p, r, _ptrs(xls), k,
                                                   _ptrs(d_a.unbind(0)), n_adapters, ptr(ws), ws_bytes, m, k, r, s),
              "lora_weight_grad_segmented")
        check(lib.qb200_lora_weight_grad_segmented(dt, n, 1, tables_p, ptr(rank_offsets), rank_total, _ptrs(us.unbind(0)), r,
                                                   _ptrs(dqs), n_out, _ptrs(d_b.unbind(0)), n_adapters, ptr(ws), ws_bytes, m,
                                                   n_out, r, s), "lora_weight_grad_segmented")
    return d_a, d_b


@dora_segmented_bwd.register_fake
def _(dqs, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dxs):
    m, n_out, k, cdt = _check_dora_bwd(dqs, tables, rank_offsets, rank_total, us, xls, ws, n_adapters, r, dxs)
    n = len(tables)
    return dqs[0].new_empty((n, rank_total * k)), dqs[0].new_empty((n, rank_total * n_out))


# ----------------------------------------------------------------------------------------------------------------------
# NF4 and 8-bit blockwise (de)quantization
# ----------------------------------------------------------------------------------------------------------------------

def _check_dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, out):
    _device(packed, absmax, code2, absmax2, offset, out)
    _check_state(absmax, code2, absmax2, offset)
    _check_blocksize(blocksize)
    if code2 is not None:
        _check_blocksize(blocksize2)
    assert packed.dtype == torch.uint8 and packed.is_contiguous(), "packed: contiguous uint8"
    if out.dtype not in DTYPE_CODE:
        raise ValueError(f"Blockwise quantization only supports 16/32-bit floats, but got {out.dtype}")
    assert out.is_contiguous(), "out must be contiguous"


def _dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, out) -> None:
    dev = out.device
    lib = _lib.load()
    F.LAUNCH_COUNTER[0] += 1
    with torch.cuda.device(dev):
        if code2 is not None:
            check(lib.qb200_dequantize_nf4_nested(ptr(packed), ptr(absmax), ptr(code2), ptr(absmax2), ptr(offset), out.numel(),
                                                  blocksize, blocksize2, ptr(out), DTYPE_CODE[out.dtype], stream_ptr(dev)),
                  "dequantize_4bit")
        else:
            check(lib.qb200_dequantize_nf4(ptr(packed), ptr(absmax), out.numel(), blocksize, ptr(out), DTYPE_CODE[out.dtype],
                                           stream_ptr(dev)), "dequantize_4bit")


@torch.library.custom_op("qlora_b200::dequantize_nf4", mutates_args=("out",))
def dequantize_nf4(packed: Tensor, absmax: Tensor, code2: Optional[Tensor], absmax2: Optional[Tensor], offset: Optional[Tensor],
                   blocksize: int, blocksize2: int, out: Tensor) -> None:
    """out = the NF4 weights of `packed` (K4; for a nested state K3 + offset add + K4 as one kernel), in out's dtype."""
    _check_dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, out)
    _dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, out)


@dequantize_nf4.register_fake
def _(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, out):
    _check_dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, out)


def _check_quantize_nf4(A, blocksize, out, absmax):
    _device(A, out, absmax)
    if A.dtype not in DTYPE_CODE:
        raise ValueError(f"Blockwise quantization only supports 16/32-bit floats, but got {A.dtype}")
    _check_blocksize(blocksize)
    assert A.is_contiguous(), "A must be contiguous"
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.numel() * 2 >= A.numel(), "out: contiguous uint8, n/2 bytes"
    assert absmax.dtype == torch.float32 and absmax.is_contiguous() and absmax.numel() * blocksize >= A.numel(), \
        "absmax: contiguous fp32, one per block"


@torch.library.custom_op("qlora_b200::quantize_nf4", mutates_args=("out", "absmax"))
def quantize_nf4(A: Tensor, blocksize: int, out: Tensor, absmax: Tensor) -> None:
    """NF4 blockwise quantization of A (K1): packed codes into `out`, the fp32 absmax of every block into `absmax`."""
    _check_quantize_nf4(A, blocksize, out, absmax)
    dev = A.device
    with torch.cuda.device(dev):
        check(_lib.load().qb200_quantize_nf4(ptr(A), DTYPE_CODE[A.dtype], A.numel(), blocksize, ptr(out), ptr(absmax),
                                             stream_ptr(dev)), "quantize_4bit")


@quantize_nf4.register_fake
def _(A, blocksize, out, absmax):
    _check_quantize_nf4(A, blocksize, out, absmax)


def _check_blockwise(code, A, absmax, blocksize, out, quantize):
    _device(code, A, absmax, out)
    _check_blocksize(blocksize)
    assert code.dtype == torch.float32 and code.is_contiguous(), "code: contiguous fp32"
    assert A.is_contiguous() and out.is_contiguous() and A.numel() == out.numel(), "A and out: contiguous, of one size"
    assert absmax.dtype == torch.float32 and absmax.is_contiguous() and absmax.numel() * blocksize >= A.numel(), \
        "absmax: contiguous fp32, one per block"
    src, dst = (A, out) if quantize else (out, A)
    assert src.dtype == torch.float32 and dst.dtype == torch.uint8, "fp32 values, uint8 codes"


@torch.library.custom_op("qlora_b200::quantize_blockwise", mutates_args=("out", "absmax"))
def quantize_blockwise(code: Tensor, A: Tensor, blocksize: int, out: Tensor, absmax: Tensor) -> None:
    """8-bit blockwise quantization of fp32 A against a 256-entry codebook (K2)."""
    _check_blockwise(code, A, absmax, blocksize, out, True)
    dev = A.device
    with torch.cuda.device(dev):
        check(_lib.load().qb200_quantize_blockwise_8bit(ptr(code), ptr(A), A.numel(), blocksize, ptr(out), ptr(absmax),
                                                        stream_ptr(dev)), "quantize_blockwise")


@quantize_blockwise.register_fake
def _(code, A, blocksize, out, absmax):
    _check_blockwise(code, A, absmax, blocksize, out, True)


@torch.library.custom_op("qlora_b200::dequantize_blockwise", mutates_args=("out",))
def dequantize_blockwise(code: Tensor, A: Tensor, absmax: Tensor, blocksize: int, out: Tensor) -> None:
    """8-bit blockwise dequantization (K3): out[i] = code[A[i]] * absmax[i // blocksize], fp32."""
    _check_blockwise(code, A, absmax, blocksize, out, False)
    dev = A.device
    with torch.cuda.device(dev):
        check(_lib.load().qb200_dequantize_blockwise_8bit(ptr(code), ptr(A), ptr(absmax), A.numel(), blocksize, ptr(out),
                                                          stream_ptr(dev)), "dequantize_blockwise")


@dequantize_blockwise.register_fake
def _(code, A, absmax, blocksize, out):
    _check_blockwise(code, A, absmax, blocksize, out, False)


# ----------------------------------------------------------------------------------------------------------------------
# DoRA: the squared row norms of a frozen NF4 weight
# ----------------------------------------------------------------------------------------------------------------------

def _check_row_norm2(packed, absmax, code2, absmax2, offset, n_out, k_in, dtype, blocksize, blocksize2):
    _check_dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, packed.new_empty(0, dtype=dtype))
    assert packed.numel() * 2 == n_out * k_in, "packed: N * K / 2 bytes"


@torch.library.custom_op("qlora_b200::weight_row_norm2", mutates_args=())
def weight_row_norm2(packed: Tensor, absmax: Tensor, code2: Optional[Tensor], absmax2: Optional[Tensor], offset: Optional[Tensor],
                     n_out: int, k_in: int, dtype: torch.dtype, blocksize: int, blocksize2: int) -> Tensor:
    """||W_f||^2 for every row f: the weight `dequantize_4bit` returns in `dtype`, squared and summed in fp32; fp32 [N]."""
    _check_row_norm2(packed, absmax, code2, absmax2, offset, n_out, k_in, dtype, blocksize, blocksize2)
    w = torch.empty((n_out, k_in), dtype=dtype, device=packed.device)
    _dequantize_nf4(packed, absmax, code2, absmax2, offset, blocksize, blocksize2, w)
    norm2 = torch.empty(n_out, dtype=torch.float32, device=w.device)
    for r0 in range(0, n_out, 2048):                       # fp32 copies of 2048 rows at a time
        norm2[r0:r0 + 2048] = w[r0:r0 + 2048].float().square().sum(1)
    return norm2


@weight_row_norm2.register_fake
def _(packed, absmax, code2, absmax2, offset, n_out, k_in, dtype, blocksize, blocksize2):
    _check_row_norm2(packed, absmax, code2, absmax2, offset, n_out, k_in, dtype, blocksize, blocksize2)
    return packed.new_empty((n_out,), dtype=torch.float32)
