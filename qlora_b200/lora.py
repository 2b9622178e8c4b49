"""Fused LoRA-over-Linear4bit (SURVEY.md 8f-1): the caller of the hot path, folded into it.

peft's `lora.Linear4bit.forward` (reached from qlora.py:386-394 `get_peft_model`) computes

    result = base(x)                                  # the NF4 GEMM
    result = result + lora_B(lora_A(dropout(x))) * scaling

i.e. two more GEMMs plus scale/add passes over [M, N] (and their mirror images in backward).  Here the low-rank
update is ONE extra bf16 contraction step of the fused kernel, accumulated in the same register accumulators:

    forward : Y  = X . W^T + U . B^T         U = scaling * (drop(X) . A^T)   [M, r]
    backward: dX = dY . W  + G . A           G = scaling * (dY . B)          [M, r]
              dA = G^T . drop(X)   dB = dY^T . U                             (the trainable adapters' grads)

Only the skinny [M, r] projections stay separate (cuBLAS).  The sum is rounded to bf16 once (the unfused
sequence rounds the base output and the update separately), so results agree with peft's to within one bf16 ulp.

Dropout (`--lora_dropout 0.1`, scripts/finetune_llama2_guanaco_7b.sh:42): the LoRA branch reads `x_lora = drop(x)`,
passed as a second input.  Forward is unchanged (U comes from x_lora); in backward the LoRA term of the input gradient
must go through the dropout mask, so it is returned as the gradient of `x_lora` (G . A, one extra skinny GEMM) and the
fused dX launch carries the base term only.

Linears that share their input and shape (q/k/v, gate/up) run as ONE grouped launch per direction
(`lora_linear4bit_group`): the three (two) forward GEMMs side by side, the backward as one long contraction
dX = sum_p (dY_p . W_p + G_p . A_p) accumulated in the same accumulators — no separate accumulation of the input gradient — and the
`x . A_p^T` projections batched into one GEMM.

fp32 activations (the reference casts its norms to fp32, qlora.py:400-401, so `Linear4bit.forward` sees fp32 in and
returns fp32): the input is cast to bf16 once per call (once per GROUP for q/k/v) and the kernel's epilogue writes the
bf16-rounded result widened to fp32 — the two output-side cast passes of `Linear4bit.forward` / its backward disappear.
"""
from __future__ import annotations

import torch

from . import functional as F


# Adapter gradients: with this switch on, dA / dB are accumulated straight into an EXISTING `.grad` buffer by the GEMM itself
# (`grad = 1 * grad + G^T . x`, cuBLAS beta = 1) and the autograd node returns None for them — one launch instead of a GEMM +
# autograd's separate `grad += new` kernel per adapter matrix (448 tiny adds per Llama-2-7B step).  Only meaningful for a
# training loop that keeps persistent `.grad` buffers and does its own gradient sync (harness/dp.py); off by default because
# hooks on the adapter gradients (DistributedDataParallel's reducer) would never fire.
ACCUMULATE_ADAPTER_GRADS_IN_PLACE = False


def _scaled_mm(a: torch.Tensor, b: torch.Tensor, scale: float, out: torch.Tensor | None = None) -> torch.Tensor:
    """scale * (a @ b) in ONE GEMM (cuBLAS alpha) — no separate scaling pass over the [M, r] projection."""
    if out is None:
        out = torch.empty((a.shape[0], b.shape[1]), dtype=a.dtype, device=a.device)
    return torch.addmm(out, a, b, beta=0.0, alpha=scale, out=out)


def _project(x2d: torch.Tensor, lora_a: torch.Tensor, scale: float) -> torch.Tensor:
    """U = scale * x2d . lora_a^T.  A decode step (<= 16 tokens) takes the library's one-launch projection, which chains with
    the skinny kernel by programmatic dependent launch; everything else is one cuBLAS GEMM."""
    if (x2d.shape[0] <= F.LORA_PROJECT_MAX_TOKENS and x2d.shape[1] % 8 == 0 and x2d.dtype == torch.bfloat16
            and lora_a.dtype == torch.bfloat16 and lora_a.is_contiguous()):
        return F.lora_project(x2d, lora_a, scale)
    return _scaled_mm(x2d, lora_a.t(), scale)


def _adapter_grad(param: torch.Tensor, a: torch.Tensor, b: torch.Tensor):
    """a @ b as the gradient of `param`: returned, or (ACCUMULATE_ADAPTER_GRADS_IN_PLACE and a grad buffer exists) added in
    place by the GEMM, in which case the node reports None."""
    g = param.grad
    if ACCUMULATE_ADAPTER_GRADS_IN_PLACE and g is not None and g.dtype == a.dtype and g.is_contiguous():
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


def _as_bf16_2d(t: torch.Tensor) -> torch.Tensor:
    t2 = t.reshape(-1, t.shape[-1])
    if t2.dtype != torch.bfloat16:
        t2 = t2.to(torch.bfloat16)
    return t2 if t2.is_contiguous() else t2.contiguous()


class LoraMatMul4Bit(torch.autograd.Function):
    """y = x . W^T + scaling * (x_lora . A^T) . B^T for ONE frozen NF4 Linear4bit (x_lora = None: the same tensor as x)."""

    @staticmethod
    def forward(ctx, x, x_lora, packed_t, lora_a, lora_b, scaling: float, quant_state: F.QuantState):
        x2d = _as_bf16_2d(x)
        xl2d = x2d if x_lora is None else _as_bf16_2d(x_lora)
        u = _project(xl2d, lora_a, scaling)
        out_dtype = torch.float32 if x.dtype == torch.float32 else torch.bfloat16
        y = F.nf4_linear_fwd_lora(x2d, packed_t, quant_state, u, lora_b.contiguous(), out_dtype=out_dtype)
        ctx.save_for_backward(xl2d, u, packed_t, lora_a, lora_b)
        ctx.adapters = (lora_a, lora_b)     # the Parameter objects themselves (their .grad buffers, see _adapter_grad)
        ctx.state = quant_state
        ctx.scaling = scaling
        ctx.x_shape = x.shape
        ctx.x_dtype = x.dtype
        ctx.split_lora = x_lora is not None
        ctx.xl_meta = None if x_lora is None else (x_lora.shape, x_lora.dtype)
        return y.view(*x.shape[:-1], quant_state.shape[0])

    @staticmethod
    def backward(ctx, grad_y):
        xl2d, u, packed_t, lora_a, lora_b = ctx.saved_tensors
        g2d = _as_bf16_2d(grad_y)
        g = _scaled_mm(g2d, lora_b, ctx.scaling)   # [M, r]
        grad_x = grad_xl = grad_a = grad_b = None
        out_dtype = torch.float32 if ctx.x_dtype == torch.float32 else torch.bfloat16
        if ctx.split_lora:
            # dropout on the LoRA branch: its input gradient goes back through the mask, the base term does not
            if ctx.needs_input_grad[0]:
                grad_x = F.nf4_linear_bwd_dx(g2d, packed_t, ctx.state, out_dtype=out_dtype).view(ctx.x_shape)
            if ctx.needs_input_grad[1]:
                shape, dtype = ctx.xl_meta
                grad_xl = torch.mm(g, lora_a).to(dtype).view(shape)
        elif ctx.needs_input_grad[0]:
            grad_x = F.nf4_linear_bwd_dx_lora(g2d, packed_t, ctx.state, g, lora_a.contiguous(), out_dtype=out_dtype).view(ctx.x_shape)
        if ctx.needs_input_grad[3]:
            grad_a = _adapter_grad(ctx.adapters[0], g.t(), xl2d)       # [r, K]
        if ctx.needs_input_grad[4]:
            grad_b = _adapter_grad(ctx.adapters[1], g2d.t(), u)        # [N, r]
        return grad_x, grad_xl, None, grad_a, grad_b, None, None


def _fusable(x, base, lora_a, lora_b) -> bool:
    qs = getattr(base.weight, "quant_state", None)
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float32) and base.bias is None and lora_a.dtype == torch.bfloat16
            and lora_b.dtype == torch.bfloat16 and qs is not None and getattr(base, "compute_dtype", None) in (None, torch.bfloat16)
            and F.lora_fused_supported(qs, torch.bfloat16, lora_a.shape[0]))


def lora_linear4bit(x: torch.Tensor, base, lora_a: torch.Tensor, lora_b: torch.Tensor, scaling: float,
                    x_lora: torch.Tensor | None = None) -> torch.Tensor:
    """`base(x) + (x_lora @ lora_a.T @ lora_b.T) * scaling` for a quantized `Linear4bit` base (no bias), fused.

    `x_lora` is the LoRA branch's input when it differs from `x` (peft applies dropout to it); None = `x`.
    Falls back to the two-step form (still on the GPU kernels) when the fused kernel does not cover the case
    (fp16 compute dtype, rank not a multiple of 8 or > 64, bias present, unsupported shape)."""
    if _fusable(x, base, lora_a, lora_b):
        return LoraMatMul4Bit.apply(x, x_lora, base.weight.t(), lora_a, lora_b, float(scaling), base.weight.quant_state)
    result = base(x)
    xl = x if x_lora is None else x_lora
    upd = torch.nn.functional.linear(torch.nn.functional.linear(xl.to(lora_a.dtype), lora_a), lora_b) * scaling
    return result + upd.to(result.dtype)


class LoraGroupMatMul4Bit(torch.autograd.Function):
    """n = 2 or 3 LoRA-wrapped Linear4bit of one shape applied to ONE input: one fused launch per direction."""

    @staticmethod
    def forward(ctx, x, scaling: float, states, n: int, *tensors):
        # tensors = x_lora[0..n) (None: no dropout), packed_t[0..n), lora_a[0..n), lora_b[0..n)
        x_loras, packeds = tensors[:n], tensors[n:2 * n]
        lora_as, lora_bs = tensors[2 * n:3 * n], tensors[3 * n:4 * n]
        x2d = _as_bf16_2d(x)
        r = lora_as[0].shape[0]
        split = x_loras[0] is not None
        if not split:   # one projection for all adapters: U_cat = scaling * x . [A_0; A_1; ..]^T
            a_cat = _adjacent_rows(lora_as)
            if a_cat is None:
                a_cat = torch.cat([a for a in lora_as], 0)
            u_cat = _project(x2d, a_cat, scaling)
            us = [u_cat[:, i * r:(i + 1) * r] for i in range(n)]
            xls = [x2d] * n
        else:
            xls = [_as_bf16_2d(t) for t in x_loras]
            us = [_project(xls[i], lora_as[i], scaling) for i in range(n)]
        out_dtype = torch.float32 if x.dtype == torch.float32 else torch.bfloat16
        ys = F.nf4_linear_group(False, [x2d] * n, list(packeds), list(states), us=us, vs=[b.contiguous() for b in lora_bs],
                                out_dtype=out_dtype)
        ctx.save_for_backward(*(xls if split else [x2d]), *us, *packeds, *lora_as, *lora_bs)
        ctx.adapters = (tuple(lora_as), tuple(lora_bs))   # the Parameter objects themselves (their .grad buffers)
        ctx.n, ctx.states, ctx.scaling, ctx.split = n, states, scaling, split
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.xl_meta = [(t.shape, t.dtype) for t in x_loras] if split else None
        n_out = states[0].shape[0]
        return tuple(y.view(*x.shape[:-1], n_out) for y in ys)

    @staticmethod
    def backward(ctx, *grad_ys):
        n, split = ctx.n, ctx.split
        saved = list(ctx.saved_tensors)
        nx = n if split else 1
        xls = saved[:nx] if split else [saved[0]] * n
        us = saved[nx:nx + n]
        packeds = saved[nx + n:nx + 2 * n]
        lora_as = saved[nx + 2 * n:nx + 3 * n]
        lora_bs = saved[nx + 3 * n:nx + 4 * n]
        g2ds = [_as_bf16_2d(g) for g in grad_ys]
        r = lora_as[0].shape[0]
        g_cat = torch.empty((g2ds[0].shape[0], n * r), dtype=torch.bfloat16, device=g2ds[0].device)
        gs = [_scaled_mm(g2ds[i], lora_bs[i], ctx.scaling, out=g_cat[:, i * r:(i + 1) * r]) for i in range(n)]   # [M, r] slices
        out_dtype = torch.float32 if ctx.x_dtype == torch.float32 else torch.bfloat16
        grad_x = None
        grad_xls = [None] * n
        if split:
            if ctx.needs_input_grad[0]:
                grad_x = F.nf4_linear_group(True, g2ds, packeds, list(ctx.states), out_dtype=out_dtype).view(ctx.x_shape)
            for i in range(n):
                if ctx.needs_input_grad[4 + i]:
                    shape, dtype = ctx.xl_meta[i]
                    grad_xls[i] = torch.mm(gs[i], lora_as[i]).to(dtype).view(shape)
        elif ctx.needs_input_grad[0]:
            # dX = sum_p (dY_p . W_p + G_p . A_p): ONE launch, one accumulator — no per-linear dX tensors, no adds
            grad_x = F.nf4_linear_group(True, g2ds, packeds, list(ctx.states), us=gs, vs=[a.contiguous() for a in lora_as],
                                        out_dtype=out_dtype).view(ctx.x_shape)
        pa, pb = ctx.adapters
        if split:
            grad_as = [_adapter_grad(pa[i], gs[i].t(), xls[i]) for i in range(n)]
        else:   # one GEMM for all adapters' dA: [G_0 | G_1 | ..]^T . x
            ga_sink = None
            if ACCUMULATE_ADAPTER_GRADS_IN_PLACE and all(a.grad is not None for a in pa):
                ga_sink = _adjacent_rows([a.grad for a in pa])
            if ga_sink is not None and ga_sink.dtype == g_cat.dtype:
                torch.addmm(ga_sink, g_cat.t(), xls[0], out=ga_sink)
                grad_as = [None] * n
            else:
                ga_cat = torch.mm(g_cat.t(), xls[0])
                grad_as = [ga_cat[i * r:(i + 1) * r] for i in range(n)]
        grad_bs = [_adapter_grad(pb[i], g2ds[i].t(), us[i]) for i in range(n)]
        return (grad_x, None, None, None, *grad_xls, *([None] * n), *grad_as, *grad_bs)


def lora_linear4bit_group(x: torch.Tensor, bases, lora_as, lora_bs, scaling: float, x_loras=None):
    """Fused `[base_p(x) + (x_lora_p @ A_p.T @ B_p.T) * scaling for p]` for 2-3 Linear4bit of one shape on one input.

    Falls back to per-linear `lora_linear4bit` calls when the group does not qualify (different shapes, bias, ...)."""
    n = len(bases)
    shapes = {tuple(b.weight.quant_state.shape) if getattr(b.weight, "quant_state", None) is not None else None for b in bases}
    ranks = {a.shape[0] for a in lora_as}
    nested = {b.weight.quant_state.nested for b in bases if getattr(b.weight, "quant_state", None) is not None}
    ok = (2 <= n <= 3 and len(shapes) == 1 and None not in shapes and len(ranks) == 1 and len(nested) == 1
          and all(_fusable(x, bases[i], lora_as[i], lora_bs[i]) for i in range(n))
          and (x_loras is None or all(t is not None for t in x_loras)))
    if not ok:
        return tuple(lora_linear4bit(x, bases[i], lora_as[i], lora_bs[i], scaling, None if x_loras is None else x_loras[i])
                     for i in range(n))
    xl = [None] * n if x_loras is None else list(x_loras)
    states = tuple(b.weight.quant_state for b in bases)
    return LoraGroupMatMul4Bit.apply(x, float(scaling), states, n, *xl, *[b.weight.t() for b in bases], *lora_as, *lora_bs)


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
    g = param.grad
    if ACCUMULATE_ADAPTER_GRADS_IN_PLACE and g is not None and g.dtype == grad.dtype and g.shape == grad.shape:
        g.add_(grad)
        return None
    return grad


class DoraMatMul4Bit(torch.autograd.Function):
    """n = 1..3 DoRA-wrapped Linear4bit of one shape applied to ONE input (q/k/v, gate/up: one launch per direction)."""

    @staticmethod
    def forward(ctx, x, scaling: float, states, n: int, *tensors):
        # tensors = x_lora[0..n) (None: no dropout), packed_t[0..n), lora_a[0..n), lora_b[0..n), magnitude[0..n)
        x_loras, packeds = tensors[:n], list(tensors[n:2 * n])
        lora_as, lora_bs, mags = tensors[2 * n:3 * n], tensors[3 * n:4 * n], tensors[4 * n:5 * n]
        states = list(states)
        x2d = _as_bf16_2d(x)
        r = lora_as[0].shape[0]
        split = x_loras[0] is not None
        norms = F.dora_weight_norm(packeds, states, list(lora_as), list(lora_bs), scaling)
        cs = [m.detach().float() / nrm for m, nrm in zip(mags, norms)]
        out_dtype = torch.float32 if x.dtype == torch.float32 else torch.bfloat16
        if not split:
            a_cat = _adjacent_rows(lora_as) if n > 1 else lora_as[0]
            if a_cat is None:
                a_cat = torch.cat(list(lora_as), 0)
            u_cat = _project(x2d, a_cat, scaling)
            us = [u_cat[:, i * r:(i + 1) * r] for i in range(n)]
            xls = [x2d] * n
            vs = [(b.float() * c[:, None]).to(torch.bfloat16) for b, c in zip(lora_bs, cs)]    # diag(c) B
            ys = F.nf4_linear_group(False, [x2d] * n, packeds, states, us=us, vs=vs, out_dtype=out_dtype, row_scales=cs)
            qs_saved = ys                                            # Q = y / c: dm = sum_t dy * y / (c n)
        else:
            xls = [_as_bf16_2d(t) for t in x_loras]
            us = [_project(xls[i], lora_as[i], scaling) for i in range(n)]
            qs_saved = F.nf4_linear_group(False, xls, packeds, states, us=us, vs=[b.contiguous() for b in lora_bs])
            ps = F.nf4_linear_group(False, [x2d - xl for xl in xls], packeds, states)
            ys = [torch.addcmul(p.float(), q.float(), c).to(out_dtype) for p, q, c in zip(ps, qs_saved, cs)]
        ctx.save_for_backward(*(xls if split else [x2d]), *us, *packeds, *lora_as, *lora_bs, *norms, *cs, *qs_saved)
        ctx.params = (tuple(lora_as), tuple(lora_bs), tuple(mags))
        ctx.n, ctx.states, ctx.scaling, ctx.split = n, states, scaling, split
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.xl_meta = [(t.shape, t.dtype) for t in x_loras] if split else None
        n_out = states[0].shape[0]
        return tuple(y.view(*x.shape[:-1], n_out) for y in ys)

    @staticmethod
    def backward(ctx, *grad_ys):
        n, split, s = ctx.n, ctx.split, ctx.scaling
        saved = list(ctx.saved_tensors)
        nx = n if split else 1
        xls = saved[:nx] if split else [saved[0]] * n
        rest = saved[nx:]
        us, packeds, lora_as, lora_bs, norms, cs, qs_saved = (rest[i * n:(i + 1) * n] for i in range(7))
        g2ds = [_as_bf16_2d(g) for g in grad_ys]
        r = lora_as[0].shape[0]
        # G_p = s (dy_p * c_p) . B_p = s dy_p . (diag(c_p) B_p), written side by side for one dA GEMM
        g_cat = torch.empty((g2ds[0].shape[0], n * r), dtype=torch.bfloat16, device=g2ds[0].device)
        gs = [_scaled_mm(g2ds[i], (lora_bs[i].float() * cs[i][:, None]).to(torch.bfloat16), s, out=g_cat[:, i * r:(i + 1) * r])
              for i in range(n)]
        out_dtype = torch.float32 if ctx.x_dtype == torch.float32 else torch.bfloat16
        grad_x = None
        grad_xls = [None] * n
        if split:
            if ctx.needs_input_grad[0]:
                grad_x = F.nf4_linear_group(True, g2ds, list(packeds), ctx.states, out_dtype=out_dtype).view(ctx.x_shape)
            for i in range(n):
                if ctx.needs_input_grad[4 + i]:
                    shape, dtype = ctx.xl_meta[i]
                    grad_xls[i] = F.nf4_linear_group(True, [g2ds[i]], [packeds[i]], [ctx.states[i]], us=[gs[i]],
                                                     vs=[lora_as[i].contiguous()], row_scales=[cs[i] - 1.0],
                                                     out_dtype=torch.float32 if dtype == torch.float32 else torch.bfloat16).view(shape)
        elif ctx.needs_input_grad[0]:
            grad_x = F.nf4_linear_group(True, g2ds, list(packeds), ctx.states, us=gs, vs=[a.contiguous() for a in lora_as],
                                        out_dtype=out_dtype, row_scales=list(cs)).view(ctx.x_shape)
        pa, pb, pm = ctx.params
        if split or n == 1:
            grad_as = [_adapter_grad(pa[i], gs[i].t(), xls[i]) for i in range(n)]
        else:
            ga_cat = torch.mm(g_cat.t(), xls[0])
            grad_as = [_accumulate_or_return(pa[i], ga_cat[i * r:(i + 1) * r]) for i in range(n)]
        grad_bs, grad_ms = [], []
        for i in range(n):
            grad_bs.append(_accumulate_or_return(pb[i], (torch.mm(g2ds[i].t(), us[i]).float() * cs[i][:, None]).to(pb[i].dtype)))
            dq = (grad_ys[i].reshape(-1, grad_ys[i].shape[-1]).float() * qs_saved[i].float()).sum(0)
            dm = dq / (norms[i] * cs[i]) if not split else dq / norms[i]
            grad_ms.append(_accumulate_or_return(pm[i], dm.to(pm[i].dtype)))
        return (grad_x, None, None, None, *grad_xls, *([None] * n), *grad_as, *grad_bs, *grad_ms)


def _dora_fusable(x, base, lora_a, lora_b, magnitude) -> bool:
    return _fusable(x, base, lora_a, lora_b) and magnitude.dtype == lora_a.dtype and magnitude.shape == (base.out_features,)


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
    if _dora_fusable(x, base, lora_a, lora_b, magnitude):
        return DoraMatMul4Bit.apply(x, float(scaling), (base.weight.quant_state,), 1, x_lora, base.weight.t(), lora_a, lora_b,
                                    magnitude)[0]
    return dora_linear4bit_peft(x, base, lora_a, lora_b, magnitude, scaling, x_lora)


def dora_linear4bit_group(x: torch.Tensor, bases, lora_as, lora_bs, magnitudes, scaling: float, x_loras=None):
    """`dora_linear4bit` for 2-3 Linear4bit of one shape on one input (q/k/v, gate/up): one launch per direction for the
    GEMMs, one launch for their weight norms.  Falls back to per-linear calls when the group does not qualify."""
    n = len(bases)
    shapes = {tuple(b.weight.quant_state.shape) if getattr(b.weight, "quant_state", None) is not None else None for b in bases}
    ranks = {a.shape[0] for a in lora_as}
    nested = {b.weight.quant_state.nested for b in bases if getattr(b.weight, "quant_state", None) is not None}
    ok = (2 <= n <= 3 and len(shapes) == 1 and None not in shapes and len(ranks) == 1 and len(nested) == 1
          and all(_dora_fusable(x, bases[i], lora_as[i], lora_bs[i], magnitudes[i]) for i in range(n))
          and (x_loras is None or all(t is not None for t in x_loras)))
    if not ok:
        return tuple(dora_linear4bit(x, bases[i], lora_as[i], lora_bs[i], magnitudes[i], scaling,
                                     None if x_loras is None else x_loras[i]) for i in range(n))
    xl = [None] * n if x_loras is None else list(x_loras)
    states = tuple(b.weight.quant_state for b in bases)
    return DoraMatMul4Bit.apply(x, float(scaling), states, n, *xl, *[b.weight.t() for b in bases], *lora_as, *lora_bs,
                                *magnitudes)
