"""Fused LoRA-over-Linear4bit (SURVEY.md 8f-1): the caller of the hot path, folded into it.

peft's `lora.Linear4bit.forward` (reached from qlora.py:386-394 `get_peft_model`) computes

    result = base(x)                                  # the NF4 GEMM
    result = result + lora_B(lora_A(dropout(x))) * scaling

i.e. two more GEMMs plus scale/add passes over [M, N] (and their mirror images in backward).  Here the low-rank
update is ONE extra 16-bit contraction step of the fused kernel, accumulated in the same register accumulators:

    forward : Y  = X . W^T + U . B^T         U = scaling * (drop(X) . A^T)   [M, r]
    backward: dX = dY . W  + G . A           G = scaling * (dY . B)          [M, r]
              dA = G^T . drop(X)   dB = dY^T . U                             (the trainable adapters' grads)

Ranks of 8..256 (multiples of 8) are one 64-wide contraction step per 64 ranks.  Only the skinny [M, r] projections stay
separate (cuBLAS).  The sum is rounded to the compute dtype once (the unfused
sequence rounds the base output and the update separately), so results agree with peft's to within one ulp of it.
The compute dtype is bf16 (over a bf16 or fp16 quant state), or fp16 for a base with `compute_dtype=torch.float16` (over an
fp16 or fp32 quant state); the adapters are of the compute dtype.  fp16 activations under bf16 compute, and fp32 states
under bf16 compute, keep the two-step form, whose base call runs fused through `Linear4bit.forward`.

Dropout (`--lora_dropout 0.1`, scripts/finetune_llama2_guanaco_7b.sh:42): the LoRA branch reads `x_lora = drop(x)`,
passed as a second input.  Forward is unchanged (U comes from x_lora); in backward the LoRA term of the input gradient
must go through the dropout mask, so it is returned as the gradient of `x_lora` (G . A, one extra skinny GEMM) and the
fused dX launch carries the base term only.

One autograd function, `LoraMatMul4Bit`, covers 1..3 linears on one input.  Linears that share their input and shape
(q/k/v, gate/up; `lora_linear4bit_group`) run as ONE grouped launch per direction: the three (two) forward GEMMs side by
side, the backward as one long contraction dX = sum_p (dY_p . W_p + G_p . A_p) accumulated in the same accumulators — no
separate accumulation of the input gradient — and the `x . A_p^T` projections batched into one GEMM.  A single linear
(`lora_linear4bit`) is the same call with one problem.

fp32 activations (the reference casts its norms to fp32, qlora.py:400-401, so `Linear4bit.forward` sees fp32 in and
returns fp32): the input is cast to the compute dtype once per call (once per GROUP for q/k/v) and the kernel's epilogue
writes the rounded result widened to fp32 — the two output-side cast passes of `Linear4bit.forward` / its backward disappear.
"""
from __future__ import annotations

import torch

from . import _ops
from . import functional as F


# Adapter gradients: with this switch on, dA / dB are accumulated straight into an EXISTING `.grad` buffer by the GEMM itself
# (`grad = 1 * grad + G^T . x`, cuBLAS beta = 1) and the autograd node returns None for them — one launch instead of a GEMM +
# autograd's separate `grad += new` kernel per adapter matrix (448 tiny adds per Llama-2-7B step).  Only meaningful for a
# training loop that keeps persistent `.grad` buffers and does its own gradient sync (harness/dp.py); off by default because
# hooks on the adapter gradients (DistributedDataParallel's reducer) would never fire.  Each forward reads the switch once and
# its backward follows that decision.  torch.compile reads it when it traces a graph; a traced backward cannot write into
# `.grad`, so leave it off for compiled models.
ACCUMULATE_ADAPTER_GRADS_IN_PLACE = False


def _scaled_mm(a: torch.Tensor, b: torch.Tensor, scale: float, out: torch.Tensor | None = None) -> torch.Tensor:
    """scale * (a @ b) in ONE GEMM (cuBLAS alpha) — no separate scaling pass over the [M, r] projection."""
    if out is None:
        out = torch.empty((a.shape[0], b.shape[1]), dtype=a.dtype, device=a.device)
    return torch.addmm(out, a, b, beta=0.0, alpha=scale, out=out)


def _project(x2d: torch.Tensor, lora_a: torch.Tensor, scale: float) -> torch.Tensor:
    """U = scale * x2d . lora_a^T (`qlora_b200::lora_project`, which picks the library's decode-step projection or cuBLAS by
    the token count at run time)."""
    if lora_a.dtype != x2d.dtype:
        return _scaled_mm(x2d, lora_a.t(), scale)
    return _ops.lora_project(x2d, lora_a, float(scale))


def _adapter_grad(param: torch.Tensor, a: torch.Tensor, b: torch.Tensor):
    """a @ b as the gradient of `param`: returned, or added in place by the GEMM when `param` is given (its forward ran with
    ACCUMULATE_ADAPTER_GRADS_IN_PLACE on; None otherwise) and has a grad buffer, in which case the node reports None."""
    g = None if param is None else param.grad
    if g is not None and g.dtype == a.dtype and g.is_contiguous():
        torch.addmm(g, a, b, out=g)
        return None
    return torch.mm(a, b)


def _adjacent_rows(ts) -> torch.Tensor | None:
    """If the 2-D tensors are consecutive row blocks of ONE contiguous buffer (the harness allocates q/k/v adapters that way),
    the [sum rows, cols] view over all of them; else None."""
    t0 = ts[0]
    if not all(t.is_contiguous() and t.shape[1] == t0.shape[1] and t.dtype == t0.dtype for t in ts):
        return None
    off = t0.storage_offset()
    for t in ts:
        if t.untyped_storage().data_ptr() != t0.untyped_storage().data_ptr() or t.storage_offset() != off:
            return None
        off += t.numel()
    rows = sum(t.shape[0] for t in ts)
    return torch.as_strided(t0.detach(), (rows, t0.shape[1]), (t0.shape[1], 1), t0.storage_offset())


def _split(seq, n: int, k: int):
    """The first k * n items of `seq` as k lists of n: the per-linear groups of an autograd function's variadic inputs, its
    saved tensors or its `needs_input_grad` flags."""
    return [list(seq[i * n:(i + 1) * n]) for i in range(k)]


def _apply(fn, x, bases, scaling: float, x_loras, *per_linear):
    """`fn.apply` on n = len(bases) linears, its variadic inputs in the order `fn.forward` splits them: x_lora[0..n) (None:
    no dropout), packed_t[0..n), then each list of `per_linear` (lora_a[0..n), lora_b[0..n), ...)."""
    n = len(bases)
    x_loras = [None] * n if x_loras is None else x_loras
    return fn.apply(x, float(scaling), tuple(b.weight.quant_state for b in bases), n, *x_loras, *[b.weight.t() for b in bases],
                    *[t for ts in per_linear for t in ts])


def _project_inputs(x2d: torch.Tensor, x_loras, lora_as, scaling: float):
    """(x_lora_p, U_p = scaling * x_lora_p . A_p^T) for every adapter, x_lora_p as [M, K] of x2d's (the compute) dtype.
    Without dropout every x_lora_p is x and ONE projection U_cat = scaling * x . [A_0; A_1; ..]^T is sliced into the U_p.  A single adapter is projected as it
    is: a cat of one non-contiguous A would be a contiguous copy, which moves a <= 16-token step onto the library's projection."""
    if x_loras[0] is not None:
        xls = [F.as_compute_2d(t, x2d.dtype) for t in x_loras]
        return xls, [_project(xl, a, scaling) for xl, a in zip(xls, lora_as)]
    n, r = len(lora_as), lora_as[0].shape[0]
    a_cat = lora_as[0] if n == 1 else _adjacent_rows(lora_as)
    if a_cat is None:
        a_cat = torch.cat(lora_as, 0)
    u_cat = _project(x2d, a_cat, scaling)
    return [x2d] * n, [u_cat[:, i * r:(i + 1) * r] for i in range(n)]


def _project_grads(g2ds, vs, scaling: float):
    """G_p = scaling * dY_p . V_p ([M, r] each), written side by side into one [M, n r] buffer G_cat for a single dA GEMM;
    returns (G_cat, [G_p])."""
    r = vs[0].shape[1]
    g_cat = torch.empty((g2ds[0].shape[0], len(vs) * r), dtype=g2ds[0].dtype, device=g2ds[0].device)
    return g_cat, [_scaled_mm(g, v, scaling, out=g_cat[:, i * r:(i + 1) * r]) for i, (g, v) in enumerate(zip(g2ds, vs))]


def _fusable(x, base, lora_a, lora_b) -> bool:
    """Whether one adapter-wrapped Linear4bit runs fused: the compute dtype is the base's fp16, else bf16 (a base with no or
    bf16 compute dtype); x is of it or fp32, the adapters of it, and the fused kernel covers the quant state and the rank."""
    qs = getattr(base.weight, "quant_state", None)
    base_cdt = getattr(base, "compute_dtype", None)
    if base_cdt not in (None, torch.bfloat16, torch.float16):
        return False
    cdt = torch.float16 if base_cdt == torch.float16 else torch.bfloat16
    # an fp32 state under bf16 compute keeps the two-step form (its base call still runs fused, through Linear4bit): fused,
    # a grouped dropout step's input gradient rounds differently from per-linear calls by more than their 4e-3 agreement bar
    return (x.is_cuda and x.dtype in (cdt, torch.float32) and base.bias is None and lora_a.dtype == cdt and lora_b.dtype == cdt
            and qs is not None and not (cdt == torch.bfloat16 and qs.dtype == torch.float32)
            and F.lora_fused_supported(qs, cdt, lora_a.shape[0]))


def _group_fusable(x, bases, lora_as, lora_bs, x_loras) -> bool:
    """Whether 1..3 adapter-wrapped Linear4bit on the input `x` run as ONE fused call: the fused kernel covers each of them,
    and they share one weight shape, one rank, one quantization form (all nested or all plain) and one rounding of the
    weights (under bf16 compute: all fp16 states or none), with a dropout input for every linear or for none."""
    if not (1 <= len(bases) <= 3 and all(_fusable(x, b, a, bb) for b, a, bb in zip(bases, lora_as, lora_bs))):
        return False
    states = [b.weight.quant_state for b in bases]
    cdt = lora_as[0].dtype
    return (len({tuple(qs.shape) for qs in states}) == 1 and len({a.shape[0] for a in lora_as}) == 1
            and len({qs.nested for qs in states}) == 1 and len({F.double_rounded(qs, cdt) for qs in states}) == 1
            and (x_loras is None or all(t is not None for t in x_loras)))


class LoraMatMul4Bit(torch.autograd.Function):
    """y_p = x . W_p^T + scaling * (x_lora_p . A_p^T) . B_p^T for n = 1..3 LoRA-wrapped Linear4bit of one shape applied to ONE
    input (q/k/v, gate/up: one fused launch per direction).  x_lora_p = None for every p: no dropout, the adapters read x.
    The adapters' dtype (bf16 or fp16) is the compute dtype."""

    @staticmethod
    def forward(ctx, x, scaling: float, states, n: int, *tensors):
        x_loras, packeds, lora_as, lora_bs = _split(tensors, n, 4)
        cdt = lora_as[0].dtype
        x2d = F.as_compute_2d(x, cdt)
        xls, us = _project_inputs(x2d, x_loras, lora_as, scaling)
        ys, scratch = F.nf4_linear_group(False, [x2d] * n, packeds, list(states), us=us, vs=[b.contiguous() for b in lora_bs],
                                         out_dtype=F.out_dtype_for(x.dtype, cdt), return_scratch=True)
        kept = F.scratch_to_save(scratch, ctx.needs_input_grad[0])   # a checkpoint recompute's W copies, for the dX launch
        ctx.save_for_backward(*xls, *us, *packeds, *lora_as, *lora_bs, *kept)
        ctx.kept_scratch = bool(kept)
        # the Parameter objects themselves, for their .grad buffers (see _adapter_grad)
        ctx.adapters = (lora_as, lora_bs) if ACCUMULATE_ADAPTER_GRADS_IN_PLACE else ([None] * n, [None] * n)
        ctx.n, ctx.states, ctx.scaling, ctx.split = n, states, scaling, x_loras[0] is not None
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.xl_meta = [(t.shape, t.dtype) for t in x_loras] if ctx.split else None
        n_out = states[0].shape[0]
        return tuple(y.view(*x.shape[:-1], n_out) for y in ys)

    @staticmethod
    def backward(ctx, *grad_ys):
        n, split = ctx.n, ctx.split
        saved = ctx.saved_tensors
        xls, us, packeds, lora_as, lora_bs = _split(saved, n, 5)
        scratch = F.saved_scratch(saved) if ctx.kept_scratch else None
        need_xl, _, need_a, need_b = _split(ctx.needs_input_grad[4:], n, 4)
        cdt = lora_as[0].dtype
        g2ds = [F.as_compute_2d(g, cdt) for g in grad_ys]
        g_cat, gs = _project_grads(g2ds, lora_bs, ctx.scaling)
        out_dtype = F.out_dtype_for(ctx.x_dtype, cdt)
        grad_x = None
        grad_xls = [None] * n
        if split:
            if ctx.needs_input_grad[0]:
                grad_x = F.nf4_linear_group(True, g2ds, packeds, list(ctx.states), out_dtype=out_dtype,
                                            w_scratch=scratch).view(ctx.x_shape)
            for i in range(n):
                if need_xl[i]:
                    shape, dtype = ctx.xl_meta[i]
                    grad_xls[i] = torch.mm(gs[i], lora_as[i]).to(dtype).view(shape)
        elif ctx.needs_input_grad[0]:
            # dX = sum_p (dY_p . W_p + G_p . A_p): ONE launch, one accumulator — no per-linear dX tensors, no adds
            grad_x = F.nf4_linear_group(True, g2ds, packeds, list(ctx.states), us=gs, vs=[a.contiguous() for a in lora_as],
                                        out_dtype=out_dtype, w_scratch=scratch).view(ctx.x_shape)
        pa, pb = ctx.adapters
        if split or n == 1:
            grad_as = [_adapter_grad(pa[i], gs[i].t(), xls[i]) if need_a[i] else None for i in range(n)]
        else:   # one GEMM for all adapters' dA: [G_0 | G_1 | ..]^T . x
            ga_sink = None
            if all(a is not None and a.grad is not None for a in pa):
                ga_sink = _adjacent_rows([a.grad for a in pa])
            if ga_sink is not None and ga_sink.dtype == g_cat.dtype:
                torch.addmm(ga_sink, g_cat.t(), xls[0], out=ga_sink)
                grad_as = [None] * n
            else:
                ga_cat = torch.mm(g_cat.t(), xls[0])
                r = lora_as[0].shape[0]
                grad_as = [ga_cat[i * r:(i + 1) * r] for i in range(n)]
        grad_bs = [_adapter_grad(pb[i], g2ds[i].t(), us[i]) if need_b[i] else None for i in range(n)]
        return (grad_x, None, None, None, *grad_xls, *([None] * n), *grad_as, *grad_bs)


def lora_linear4bit(x: torch.Tensor, base, lora_a: torch.Tensor, lora_b: torch.Tensor, scaling: float,
                    x_lora: torch.Tensor | None = None) -> torch.Tensor:
    """`base(x) + (x_lora @ lora_a.T @ lora_b.T) * scaling` for a quantized `Linear4bit` base (no bias), fused.

    `x_lora` is the LoRA branch's input when it differs from `x` (peft applies dropout to it); None = `x`.
    Falls back to the two-step form (still on the GPU kernels) when the fused kernel does not cover the case
    (fp32 compute dtype, rank not a multiple of 8 or > 256, bias present, unsupported shape or quant-state dtype)."""
    x_loras = None if x_lora is None else [x_lora]
    if _group_fusable(x, [base], [lora_a], [lora_b], x_loras):
        return _apply(LoraMatMul4Bit, x, [base], scaling, x_loras, [lora_a], [lora_b])[0]
    result = base(x)
    xl = x if x_lora is None else x_lora
    upd = torch.nn.functional.linear(torch.nn.functional.linear(xl.to(lora_a.dtype), lora_a), lora_b) * scaling
    return result + upd.to(result.dtype)


def lora_linear4bit_group(x: torch.Tensor, bases, lora_as, lora_bs, scaling: float, x_loras=None):
    """Fused `[base_p(x) + (x_lora_p @ A_p.T @ B_p.T) * scaling for p]` for 1-3 Linear4bit of one shape on one input.

    Falls back to per-linear `lora_linear4bit` calls when the group does not qualify (different shapes, bias, ...)."""
    if not _group_fusable(x, bases, lora_as, lora_bs, x_loras):
        return tuple(lora_linear4bit(x, bases[i], lora_as[i], lora_bs[i], scaling, None if x_loras is None else x_loras[i])
                     for i in range(len(bases)))
    return _apply(LoraMatMul4Bit, x, bases, scaling, x_loras, lora_as, lora_bs)


# ----------------------------------------------------------------------------------------------------------------------
# DoRA over the NF4 base ("QDoRA"; Liu et al., ICML 2024; peft `use_dora=True` on a Linear4bit)
# ----------------------------------------------------------------------------------------------------------------------
# With the detached weight norm n = ||W + s.B.A||_row and c = m / n (fp32), peft's DoraLinearLayer computes
#     no dropout : y = c * (x . W^T + s (x . A^T) . B^T)
#     dropout    : y = x . W^T + (c - 1) * (xd . W^T) + c * s (xd . A^T) . B^T,    xd = drop(x)
# A per-output-feature scale of W is a scale of the absmax of every NF4 block of that row, so the kernels take c as a row
# scale: no dropout is ONE fused launch  y = x . (diag(c) W)^T + U . (diag(c) B)^T;  with dropout
# y = (x - xd) . W^T + c * Q,  Q = xd . W^T + U . B^T  (one fused LoRA launch + one plain launch).  Backward:
#     dQ = dy * c,  G = s dQ . B = s dy . (diag(c) B),  dA = G^T . xd,  dB = dQ^T . U,  dm = sum_t dy * Q / n
#     no dropout : dx  = dy . diag(c) W + G . A                           (one launch, row scale c)
#     dropout    : dx  = dy . W,   dxd = dy . diag(c - 1) W + G . A      (row scale c - 1; dxd flows back through the mask)


def _accumulate_or_return(param: torch.Tensor, grad: torch.Tensor):
    """`grad` as the gradient of `param`, or added in place to its existing buffer (see ACCUMULATE_ADAPTER_GRADS_IN_PLACE)."""
    g = None if param is None else param.grad
    if g is not None and g.dtype == grad.dtype and g.shape == grad.shape:
        g.add_(grad)
        return None
    return grad


class DoraMatMul4Bit(torch.autograd.Function):
    """n = 1..3 DoRA-wrapped Linear4bit of one shape applied to ONE input (q/k/v, gate/up: one launch per direction)."""

    @staticmethod
    def forward(ctx, x, scaling: float, states, n: int, *tensors):
        x_loras, packeds, lora_as, lora_bs, mags = _split(tensors, n, 5)
        states = list(states)
        x2d = F.as_compute_2d(x)
        split = x_loras[0] is not None
        norms = F.dora_weight_norm(packeds, states, lora_as, lora_bs, scaling)
        cs = [m.detach().float() / nrm for m, nrm in zip(mags, norms)]
        out_dtype = F.out_dtype_for(x.dtype)
        xls, us = _project_inputs(x2d, x_loras, lora_as, scaling)
        if not split:
            vs = [(b.float() * c[:, None]).to(torch.bfloat16) for b, c in zip(lora_bs, cs)]    # diag(c) B
            ys = F.nf4_linear_group(False, [x2d] * n, packeds, states, us=us, vs=vs, out_dtype=out_dtype, row_scales=cs)
            qs_saved = ys                                            # Q = y / c: dm = sum_t dy * y / (c n)
        else:
            qs_saved = F.nf4_linear_group(False, xls, packeds, states, us=us, vs=[b.contiguous() for b in lora_bs])
            ps = F.nf4_linear_group(False, [x2d - xl for xl in xls], packeds, states)
            ys = [torch.addcmul(p.float(), q.float(), c).to(out_dtype) for p, q, c in zip(ps, qs_saved, cs)]
        ctx.save_for_backward(*xls, *us, *packeds, *lora_as, *lora_bs, *norms, *cs, *qs_saved)
        ctx.params = (lora_as, lora_bs, mags) if ACCUMULATE_ADAPTER_GRADS_IN_PLACE else ([None] * n,) * 3
        ctx.mag_dtypes = [m.dtype for m in mags]
        ctx.n, ctx.states, ctx.scaling, ctx.split = n, states, scaling, split
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.xl_meta = [(t.shape, t.dtype) for t in x_loras] if split else None
        n_out = states[0].shape[0]
        return tuple(y.view(*x.shape[:-1], n_out) for y in ys)

    @staticmethod
    def backward(ctx, *grad_ys):
        n, split, s = ctx.n, ctx.split, ctx.scaling
        xls, us, packeds, lora_as, lora_bs, norms, cs, qs_saved = _split(ctx.saved_tensors, n, 8)
        need_xl = ctx.needs_input_grad[4:4 + n]
        g2ds = [F.as_compute_2d(g) for g in grad_ys]
        # G_p = s (dy_p * c_p) . B_p = s dy_p . (diag(c_p) B_p)
        g_cat, gs = _project_grads(g2ds, [(b.float() * c[:, None]).to(torch.bfloat16) for b, c in zip(lora_bs, cs)], s)
        out_dtype = F.out_dtype_for(ctx.x_dtype)
        grad_x = None
        grad_xls = [None] * n
        if split:
            if ctx.needs_input_grad[0]:
                grad_x = F.nf4_linear_group(True, g2ds, packeds, ctx.states, out_dtype=out_dtype).view(ctx.x_shape)
            for i in range(n):
                if need_xl[i]:
                    shape, dtype = ctx.xl_meta[i]
                    grad_xls[i] = F.nf4_linear_group(True, [g2ds[i]], [packeds[i]], [ctx.states[i]], us=[gs[i]],
                                                     vs=[lora_as[i].contiguous()], row_scales=[cs[i] - 1.0],
                                                     out_dtype=F.out_dtype_for(dtype)).view(shape)
        elif ctx.needs_input_grad[0]:
            grad_x = F.nf4_linear_group(True, g2ds, packeds, ctx.states, us=gs, vs=[a.contiguous() for a in lora_as],
                                        out_dtype=out_dtype, row_scales=cs).view(ctx.x_shape)
        pa, pb, pm = ctx.params
        if split or n == 1:
            grad_as = [_adapter_grad(pa[i], gs[i].t(), xls[i]) for i in range(n)]
        else:
            r = lora_as[0].shape[0]
            ga_cat = torch.mm(g_cat.t(), xls[0])
            grad_as = [_accumulate_or_return(pa[i], ga_cat[i * r:(i + 1) * r]) for i in range(n)]
        grad_bs, grad_ms = [], []
        for i in range(n):
            grad_bs.append(_accumulate_or_return(pb[i], (torch.mm(g2ds[i].t(), us[i]).float() * cs[i][:, None]).to(lora_bs[i].dtype)))
            dq = (grad_ys[i].reshape(-1, grad_ys[i].shape[-1]).float() * qs_saved[i].float()).sum(0)
            dm = dq / (norms[i] * cs[i]) if not split else dq / norms[i]
            grad_ms.append(_accumulate_or_return(pm[i], dm.to(ctx.mag_dtypes[i])))
        return (grad_x, None, None, None, *grad_xls, *([None] * n), *grad_as, *grad_bs, *grad_ms)


def _dora_fusable(x, bases, lora_as, lora_bs, magnitudes, x_loras) -> bool:
    # bf16 compute over bf16 states only: fp16 DoRA, and DoRA over an fp16 or fp32 state, take the peft form
    return (all(a.dtype == torch.bfloat16 for a in lora_as) and _group_fusable(x, bases, lora_as, lora_bs, x_loras)
            and all(b.weight.quant_state.dtype == torch.bfloat16 for b in bases)
            and all(m.dtype == a.dtype and m.shape == (b.out_features,) for b, a, m in zip(bases, lora_as, magnitudes)))


def dora_linear4bit_peft(x, base, lora_a, lora_b, magnitude, scaling: float, x_lora=None):
    """peft's `lora.Linear` + `DoraLinearLayer` forward for a Linear4bit base, restated on the library's unfused kernels:
    the whole NF4 weight is dequantized every call for the norm and, with dropout, the base GEMM runs a second time on the
    dropped input.  The reference the fused path is checked and timed against, and its fallback."""
    result = base(x)
    weight = F.dequantize_4bit(base.weight.data, base.weight.quant_state).to(lora_a.dtype)
    lora_weight = lora_b @ lora_a
    weight_norm = torch.linalg.norm(weight + scaling * lora_weight.detach(), dim=1).to(weight.dtype).detach()
    mag_norm_scale = (magnitude / weight_norm).view(1, -1)
    xl = x if x_lora is None else x_lora
    xl = xl.to(lora_a.dtype)
    lora_result = torch.nn.functional.linear(torch.nn.functional.linear(xl, lora_a), lora_b)
    if x_lora is None:
        base_result = result if base.bias is None else result - base.bias
    else:
        base_result = torch.nn.functional.linear(xl, weight)
    result_dora = (mag_norm_scale - 1) * base_result + mag_norm_scale * lora_result * scaling
    return result + result_dora.to(result.dtype)


def dora_linear4bit(x: torch.Tensor, base, lora_a: torch.Tensor, lora_b: torch.Tensor, magnitude: torch.Tensor, scaling: float,
                    x_lora: torch.Tensor | None = None) -> torch.Tensor:
    """DoRA over a quantized `Linear4bit` base (peft `use_dora=True`), fused: the magnitude `m` rescales the rows of W inside
    the NF4 kernels.  `x_lora` is the dropped input of the adapter branch (None: no dropout / eval).  Falls back to
    `dora_linear4bit_peft` where `lora_linear4bit` falls back (rank, bias, dtype, shape)."""
    x_loras = None if x_lora is None else [x_lora]
    if _dora_fusable(x, [base], [lora_a], [lora_b], [magnitude], x_loras):
        return _apply(DoraMatMul4Bit, x, [base], scaling, x_loras, [lora_a], [lora_b], [magnitude])[0]
    return dora_linear4bit_peft(x, base, lora_a, lora_b, magnitude, scaling, x_lora)


def dora_linear4bit_group(x: torch.Tensor, bases, lora_as, lora_bs, magnitudes, scaling: float, x_loras=None):
    """`dora_linear4bit` for 1-3 Linear4bit of one shape on one input (q/k/v, gate/up): one launch per direction for the
    GEMMs, one launch for their weight norms.  Falls back to per-linear calls when the group does not qualify."""
    if not _dora_fusable(x, bases, lora_as, lora_bs, magnitudes, x_loras):
        return tuple(dora_linear4bit(x, bases[i], lora_as[i], lora_bs[i], magnitudes[i], scaling,
                                     None if x_loras is None else x_loras[i]) for i in range(len(bases)))
    return _apply(DoraMatMul4Bit, x, bases, scaling, x_loras, lora_as, lora_bs, magnitudes)
