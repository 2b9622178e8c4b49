"""Mixed-adapter batches over the NF4 base: each token row uses its own LoRA adapter (peft's `adapter_names`).

peft's `_mixed_batch_forward` computes the base forward once, then for every adapter in the batch gathers its rows, runs
`lora_B(lora_A(x_rows)) * scaling` and adds the result back: five small launches per adapter and linear.  Here, for row t
with adapter a(t) (none for "__base__"):

    y_t = x_t . W^T (+ bias) + [a(t) present] . U_t . B_a^T,      U_t = s_a . x_t . A_a^T  (rounded once to the compute dtype)

with the sum rounded once, as `lora_linear4bit` does, except on the segmented path below.

* Decode (at most `DECODE_MAX_TOKENS` rows): one `lora_project_mixed` launch per linear writes U [M, R] (each row its own
  adapter's A and scale from a device table, zero beyond its rank and for base rows), then one skinny launch per linear whose
  epilogue reads row n of each token's own B.  No host branch depends on which adapters the batch uses, so a captured CUDA
  graph switches requests by a copy into the row-index buffer (`LoraAdapterSet.indices(names, out=buffer)`).
* Above `DECODE_MAX_TOKENS` rows, the row-index tensor form takes the segmented path at every token count: the base launch
  without LoRA operands, then `lora_segmented_add`, which groups the rows by adapter on the device and adds each row's own
  U . B_a^T in place with tensor-core kernels.  No host branch depends on the indices and nothing is read back to the host,
  so such a batch too can be captured in a CUDA graph or compiled.  It rounds twice: the base output (`Linear4bit`'s bits,
  which rows without an adapter keep), then the sum.
* The names form above `DECODE_MAX_TOKENS` rows picks its branch from the names on the host (`prefill_branch`).  When the
  ranks of the adapters present add up to at most 256 ("concat"): their B matrices side by side are one V [N, sum r],
  U [M, sum r] keeps in each row only its own adapter's block, and one existing fused (or scratch) LoRA launch runs, with
  one rounding.  Otherwise ("grouped"): the adapters present are split into groups of at most 256 ranks, and the rows of
  each group run that concat launch on their own, so each NF4 weight is read once per group; one rounding too.  The names
  form keeps one rounding because, under bf16 compute, the segmented path's two roundings exceed the Frobenius-relative
  1e-3 bar against float64 that `lora_linear4bit` meets (2.3e-3 measured at 1600 rows); every element stays within 1 ulp.

Inference only, as in peft: a call in grad mode with an input or adapter weight that requires grad raises.  Dropout is the
identity.  Training takes `lora_linear4bit_group_multi` / `lora_linear4bit_multi` (end of this file): the segmented forward
at every token count, differentiable in the input and every adapter's weights (DESIGN.md §6d).  DoRA adapters
(`DoraAdapterSet`) train through `dora_linear4bit_group_multi` / `dora_linear4bit_multi` (DESIGN.md §6e).  The compute dtype is the base's (bf16, or fp16 for `compute_dtype=torch.float16`) over the quant states the fused
path covers; the adapters are of it.
"""
from __future__ import annotations

from typing import Sequence, Union

import torch
from torch import Tensor

from . import _lib, _ops
from . import functional as F

BASE_NAME = "__base__"
DECODE_MAX_TOKENS = F.LORA_PROJECT_MAX_TOKENS


class LoraAdapterSet:
    """The adapters of one linear, `{name: (lora_A.weight [r, K], lora_B.weight [N, r], scaling)}`, built once.

    Owns the device table the kernels read (one `qb200_lora_adapter` per adapter: pointers to A and B, scale, rank) and keeps
    references to the weights, so no call copies them.  The table holds the weights' addresses: rebuild the set after
    replacing a weight's storage.  Ranks are multiples of 8 in [8, 256] and may differ between adapters."""

    def __init__(self, adapters: dict):
        if not adapters:
            raise ValueError("LoraAdapterSet: no adapters")
        if BASE_NAME in adapters:
            raise ValueError(f"LoraAdapterSet: {BASE_NAME!r} names the base rows, not an adapter")
        self.names = list(adapters)
        self.index = {name: i for i, name in enumerate(self.names)}
        self.lora_as, self.lora_bs, self.scales, self.ranks = [], [], [], []
        a0 = next(iter(adapters.values()))[0]
        self.dtype, self.device = a0.dtype, a0.device
        self.in_features = a0.shape[1]
        self.out_features = next(iter(adapters.values()))[1].shape[0]
        if self.dtype not in (torch.bfloat16, torch.float16) or not a0.is_cuda:
            raise ValueError("LoraAdapterSet: bf16 or fp16 adapters on a CUDA device")
        entries = (_lib.LoraAdapter * len(self.names))()
        for i, (name, (a, b, scaling)) in enumerate(adapters.items()):
            r = a.shape[0]
            if a.dim() != 2 or b.dim() != 2 or a.shape[1] != self.in_features or b.shape != (self.out_features, r):
                raise ValueError(f"adapter {name!r}: lora_A [r, {self.in_features}] and lora_B [{self.out_features}, r]")
            if not (8 <= r <= F.LORA_MAX_RANK and r % 8 == 0):
                raise ValueError(f"adapter {name!r}: rank {r} is not a multiple of 8 in [8, {F.LORA_MAX_RANK}]")
            for t in (a, b):
                if t.dtype != self.dtype or t.device != self.device or not t.is_contiguous() or t.data_ptr() % 16:
                    raise ValueError(f"adapter {name!r}: contiguous, 16-byte aligned {self.dtype} weights on {self.device}")
            self.lora_as.append(a)
            self.lora_bs.append(b)
            self.scales.append(float(scaling))
            self.ranks.append(r)
            entries[i] = _lib.LoraAdapter(a.data_ptr(), b.data_ptr(), float(scaling), r)
        self.rmax = max(self.ranks)
        self.table = torch.frombuffer(bytearray(bytes(entries)), dtype=torch.uint8).to(self.device)
        # adapter a's rows in the flat weight-gradient buffers of `lora_linear4bit_group_multi`: [offsets[a], offsets[a] + r_a)
        offsets = [sum(self.ranks[:i]) for i in range(len(self.ranks))]
        self.rank_offsets_host = offsets
        self.rank_total = sum(self.ranks)
        self.rank_offsets = torch.tensor(offsets, dtype=torch.int64).to(self.device)

    def __len__(self) -> int:
        return len(self.names)

    def indices(self, adapter_names: Sequence[str], out: Tensor | None = None) -> Tensor:
        """The int32 row-index tensor of `adapter_names` (-1 for "__base__") on the adapters' device, or copied into `out` (a
        CUDA graph's index buffer).  An unknown name raises ValueError, as in peft."""
        unknown = sorted({n for n in adapter_names if n != BASE_NAME and n not in self.index})
        if unknown:
            raise ValueError(f"Trying to infer with non-existing adapter(s): {', '.join(unknown)}")
        idx = torch.tensor([self.index.get(n, -1) for n in adapter_names], dtype=torch.int32)
        if out is None:
            return idx.to(self.device)
        return out.copy_(idx, non_blocking=False)

    def requires_grad(self) -> bool:
        return any(t.requires_grad for t in self.lora_as + self.lora_bs)


def _compute_dtype(base) -> torch.dtype:
    return torch.float16 if getattr(base, "compute_dtype", None) == torch.float16 else torch.bfloat16


def _validate(x: Tensor, bases, sets, training: bool = False) -> torch.dtype:
    if not (1 <= len(bases) <= 3 and len(sets) == len(bases)):
        raise ValueError("1..3 Linear4bit bases with one LoraAdapterSet each")
    if not training and torch.is_grad_enabled() and (x.requires_grad or any(s.requires_grad() for s in sets)):
        raise RuntimeError("mixed-adapter batches are inference only (peft refuses adapter_names in training mode): call under "
                           "torch.no_grad() or torch.inference_mode()")
    cdt = _compute_dtype(bases[0])
    shape = tuple(bases[0].weight.quant_state.shape)
    for base, s in zip(bases, sets):
        qs = base.weight.quant_state
        if _compute_dtype(base) != cdt or tuple(qs.shape) != shape or not F.fused_supported(qs, cdt):
            raise ValueError("mixed-adapter batches: bases of one shape and compute dtype whose quant states the fused "
                             "kernels cover")
        if s.dtype != cdt or (s.out_features, s.in_features) != shape:
            raise ValueError(f"adapter set: {cdt} adapters of the base's shape")
        if s.names != sets[0].names:
            raise ValueError("grouped adapter sets must hold the same adapter names in the same order")
    states = [b.weight.quant_state for b in bases]
    if len({qs.nested for qs in states}) != 1 or len({F.double_rounded(qs, cdt) for qs in states}) != 1:
        raise ValueError("grouped bases must share their quantization form and quant-state rounding")
    if not (x.is_cuda and x.dtype in (cdt, torch.float32) + ((torch.float16,) if cdt == torch.bfloat16 else ())):
        raise ValueError(f"x: a CUDA tensor of {cdt} or float32")
    return cdt


def _bias(base, cdt):
    return None if base.bias is None else base.bias.to(cdt)


def _decode(x2d: Tensor, bases, sets, rows: Tensor, cdt):
    r = max(s.rmax for s in sets)
    us = [_ops.lora_project_mixed(x2d, s.table, rows, len(s), r) for s in sets]
    states = [b.weight.quant_state for b in bases]
    sts = [F._state_tensors(qs, x2d.device) for qs in states]
    n_out, k_in = states[0].shape
    outs = [torch.empty((x2d.shape[0], n_out), dtype=cdt, device=x2d.device) for _ in bases]
    _ops.nf4_linear_group_mixed(x2d, [b.weight.t() for b in bases], [a_f32 if a_u8 is None else a_u8 for a_u8, _, _, _, a_f32 in sts],
                                [t[1] for t in sts], [t[2] for t in sts], [t[3] for t in sts], n_out, k_in, states[0].dtype,
                                [_bias(b, cdt) for b in bases], us, [s.table for s in sets], rows, len(sets[0]), outs)
    return outs


def _concat_u(x2d: Tensor, s: LoraAdapterSet, present, rows: Tensor) -> Tensor:
    """U [M, sum r]: row t keeps only the block of its own adapter (scaled, rounded once), zero elsewhere."""
    if len(present) == 1:
        a = present[0]
        u = _ops.lora_project(x2d, s.lora_as[a], s.scales[a])   # lora_linear4bit's projection, bit for bit
        return torch.where((rows == a)[:, None], u, torch.zeros((), dtype=u.dtype, device=u.device))
    total = sum(s.ranks[a] for a in present)
    u = torch.empty((x2d.shape[0], total), dtype=x2d.dtype, device=x2d.device)
    lo = torch.full((len(s),), total, dtype=torch.int64)
    c = 0
    for a in present:   # one GEMM per adapter present, its scale as alpha: U is rounded once
        torch.addmm(u[:, c:c + s.ranks[a]], x2d, s.lora_as[a].t(), beta=0.0, alpha=s.scales[a], out=u[:, c:c + s.ranks[a]])
        lo[a] = c
        c += s.ranks[a]
    ranks = torch.tensor(s.ranks, dtype=torch.int64)
    lo_d, hi_d = lo.to(x2d.device), (lo + ranks).to(x2d.device)
    safe = rows.clamp(0, len(s) - 1).long()
    row_lo = torch.where(rows >= 0, lo_d[safe], total)
    row_hi = torch.where(rows >= 0, hi_d[safe], total)
    col = torch.arange(total, device=x2d.device)
    keep = (col[None, :] >= row_lo[:, None]) & (col[None, :] < row_hi[:, None])
    return torch.where(keep, u, torch.zeros((), dtype=u.dtype, device=u.device))


def _base_outs(x2d: Tensor, bases, cdt):
    return F.nf4_linear_group(False, [x2d] * len(bases), [b.weight.t() for b in bases], [b.weight.quant_state for b in bases],
                              biases=[_bias(b, cdt) for b in bases])


def _segmented(x2d: Tensor, bases, sets, rows: Tensor, cdt):
    outs = _base_outs(x2d, bases, cdt)
    _ops.lora_segmented_add(x2d, [s.table for s in sets], rows, len(sets[0]), max(s.rmax for s in sets), outs)
    return outs


def _rank_groups(sets, present):
    """The adapters present split, in index order, into groups whose ranks add up to at most 256 in every set."""
    groups, cur = [], []
    for a in present:
        if cur and any(sum(s.ranks[b] for b in cur) + s.ranks[a] > F.LORA_MAX_RANK for s in sets):
            groups.append(cur)
            cur = []
        cur.append(a)
    return groups + [cur]


def _grouped(x2d: Tensor, bases, sets, rows: Tensor, names, cdt):
    """Σr > 256: the adapters present in groups of at most 256 ranks; the rows of each group (known on the host from the
    names) through one concat launch, the base rows through the plain base.  One rounding per row, as the concat branch;
    each NF4 weight is read once per group rather than once per adapter."""
    index = sets[0].index
    by_adapter = {}
    for t, name in enumerate(names):
        by_adapter.setdefault(index.get(name, -1), []).append(t)
    outs = [torch.empty((x2d.shape[0], s.out_features), dtype=cdt, device=x2d.device) for s in sets]
    present = sorted(a for a in by_adapter if a >= 0)
    for group in _rank_groups(sets, present) + ([None] if -1 in by_adapter else []):
        ts = by_adapter[-1] if group is None else sorted(t for a in group for t in by_adapter[a])
        idx = torch.tensor(ts, dtype=torch.long).to(x2d.device)
        xg = x2d.index_select(0, idx)
        ys = _base_outs(xg, bases, cdt) if group is None else _concat(xg, bases, sets, rows.index_select(0, idx), group, cdt)
        for out, y in zip(outs, ys):
            out.index_copy_(0, idx, y)
    return outs


def _concat(x2d: Tensor, bases, sets, rows: Tensor, present, cdt):
    if not present:
        return _base_outs(x2d, bases, cdt)
    states = [b.weight.quant_state for b in bases]
    packeds = [b.weight.t() for b in bases]
    biases = [_bias(b, cdt) for b in bases]
    us = [_concat_u(x2d, s, present, rows) for s in sets]
    vs = [s.lora_bs[present[0]] if len(present) == 1 else torch.cat([s.lora_bs[a] for a in present], 1) for s in sets]
    if len({u.shape[1] for u in us}) == 1:
        return F.nf4_linear_group(False, [x2d] * len(bases), packeds, states, biases=biases, us=us, vs=vs)
    return [F.nf4_linear_group(False, [x2d], [p], [qs], biases=[b], us=[u], vs=[v])[0]
            for p, qs, b, u, v in zip(packeds, states, biases, us, vs)]


def prefill_branch(sets, adapter_names: Sequence[str]) -> str:
    """Which branch a batch of names takes above `DECODE_MAX_TOKENS` rows: "concat" (ranks of the adapters present add up to
    at most 256, or no adapter present) or "grouped" (the rows grouped by adapter, one concat launch per 256 ranks)."""
    present = {n for n in adapter_names if n != BASE_NAME}
    for s in sets:
        if sum(s.ranks[s.index[n]] for n in present) > F.LORA_MAX_RANK:
            return "grouped"
    return "concat"


def lora_linear4bit_group_mixed(x: Tensor, bases, adapter_sets, adapter_names: Union[Sequence[str], Tensor]):
    """`[base_p(x) + per-row LoRA of adapter_sets[p]]` for 1..3 Linear4bit of one shape on one input (q/k/v, gate/up), each
    row of `x` (flattened to [M, K]) with its own adapter.  `adapter_names`: one name per row ("__base__": no adapter), as
    peft's `adapter_names`, or the int32 CUDA row-index tensor of `LoraAdapterSet.indices` (what a CUDA graph or a compiled
    graph takes; an index outside [0, len(set)) means no adapter).  Returns a tuple of outputs of x's shape[:-1] + [N]."""
    _refuse_dora(adapter_sets)
    cdt = _validate(x, bases, adapter_sets)
    x2d = F.as_compute_2d(x, cdt)
    m = x2d.shape[0]
    if isinstance(adapter_names, Tensor):
        rows = adapter_names
        if rows.dtype != torch.int32 or rows.shape != (m,) or rows.device != x2d.device:
            raise ValueError(f"row indices: int32 [{m}] on {x2d.device}")
    else:
        if len(adapter_names) != m:
            raise ValueError(f"adapter_names: one name per row, {m} rows, got {len(adapter_names)}")
        rows = adapter_sets[0].indices(adapter_names)
    rows = rows if rows.is_contiguous() else rows.contiguous()
    if m <= DECODE_MAX_TOKENS:
        ys = _decode(x2d, bases, adapter_sets, rows, cdt)
    elif isinstance(adapter_names, Tensor):
        ys = _segmented(x2d, bases, adapter_sets, rows, cdt)
    elif prefill_branch(adapter_sets, adapter_names) == "concat":
        present = sorted({adapter_sets[0].index[n] for n in adapter_names if n != BASE_NAME})
        ys = _concat(x2d, bases, adapter_sets, rows, present, cdt)
    else:
        ys = _grouped(x2d, bases, adapter_sets, rows, adapter_names, cdt)
    out_dtype = F.out_dtype_for(x.dtype, cdt)
    n_out = bases[0].weight.quant_state.shape[0]
    return tuple((y if y.dtype == out_dtype else y.to(out_dtype)).view(*x.shape[:-1], n_out) for y in ys)


def lora_linear4bit_mixed(x: Tensor, base, adapters: LoraAdapterSet, adapter_names: Union[Sequence[str], Tensor]) -> Tensor:
    """`base(x)` plus, for every row of x, the LoRA update of its own adapter in `adapters` (peft's mixed batch forward for
    one Linear4bit).  See `lora_linear4bit_group_mixed`."""
    return lora_linear4bit_group_mixed(x, [base], [adapters], adapter_names)[0]


# ----------------------------------------------------------------------------------------------------------------------
# training several adapters over one base in one batch (DESIGN.md §6d)
# ----------------------------------------------------------------------------------------------------------------------

class MultiLoraMatMul4Bit(torch.autograd.Function):
    """y_p[t] = x[t] . W_p^T (+bias_p) + U_p[t] . B_{p,a}^T with U_p[t] = rn(s_{p,a} . xl_p[t] . A_{p,a}^T), a = rows[t], for
    n = 1..3 Linear4bit of one shape on one input; xl_p = x without dropout.  The forward is the segmented forward of
    `lora_linear4bit_group_mixed` (`lora_segmented_fwd`, which also returns U and the segment table); the backward is
    the base dX launch plus `lora_segmented_bwd`.  Differentiable in x, the dropped inputs and every adapter's A and B."""

    @staticmethod
    def forward(ctx, x, rows, states, sets, n: int, *tensors):
        x_loras, packeds, biases = (list(tensors[i * n:(i + 1) * n]) for i in range(3))
        cdt = sets[0].dtype
        x2d = F.as_compute_2d(x, cdt)
        split = x_loras[0] is not None
        xls = [F.as_compute_2d(t, cdt) for t in x_loras] if split else [x2d]
        outs = F.nf4_linear_group(False, [x2d] * n, packeds, list(states), biases=biases)
        r = max(s.rmax for s in sets)
        us, ws = _ops.lora_segmented_fwd(xls, [s.table for s in sets], rows, len(sets[0]), r, outs)
        ctx.save_for_backward(us, ws, *xls, *packeds)
        ctx.n, ctx.states, ctx.sets, ctx.r, ctx.split = n, states, sets, r, split
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.xl_meta = [(t.shape, t.dtype) for t in x_loras] if split else None
        out_dtype = F.out_dtype_for(x.dtype, cdt)
        n_out = states[0].shape[0]
        return tuple((y if y.dtype == out_dtype else y.to(out_dtype)).view(*x.shape[:-1], n_out) for y in outs)

    @staticmethod
    def backward(ctx, *grad_ys):
        n, sets, split = ctx.n, ctx.sets, ctx.split
        us, ws, *rest = ctx.saved_tensors
        xls, packeds = rest[:len(rest) - n], rest[len(rest) - n:]
        need = ctx.needs_input_grad
        need_xl = need[5:5 + n]
        n_ad = len(sets[0])
        cdt = sets[0].dtype
        g2ds = [F.as_compute_2d(g, cdt) for g in grad_ys]
        dx = F.nf4_linear_group(True, g2ds, packeds, list(ctx.states), out_dtype=cdt) if need[0] else None
        # without dropout the adapters' input-gradient term is added in place to the base dX; with it, to each dropped input
        dxl, d_a, d_b = _ops.lora_segmented_bwd(g2ds, [s.table for s in sets], sets[0].rank_offsets, sets[0].rank_total, us,
                                                list(xls), ws, n_ad, ctx.r, None if split else dx, split)
        grad_x = None if dx is None else dx.to(ctx.x_dtype).view(ctx.x_shape)
        grad_xls = [None] * n
        if split:
            for p in range(n):
                if need_xl[p]:
                    shape, dtype = ctx.xl_meta[p]
                    grad_xls[p] = dxl[p].to(dtype).view(shape)
        k, n_out = xls[0].shape[1], g2ds[0].shape[1]
        offs, ranks = sets[0].rank_offsets_host, sets[0].ranks
        base = 5 + 3 * n
        grad_as = [d_a[p, offs[a] * k:(offs[a] + ranks[a]) * k].view(ranks[a], k) if need[base + p * n_ad + a] else None
                   for p in range(n) for a in range(n_ad)]
        base += n * n_ad
        grad_bs = [d_b[p, offs[a] * n_out:(offs[a] + ranks[a]) * n_out].view(n_out, ranks[a]) if need[base + p * n_ad + a] else None
                   for p in range(n) for a in range(n_ad)]
        return (grad_x, None, None, None, None, *grad_xls, *([None] * 2 * n), *grad_as, *grad_bs)


def _rows_tensor(rows, sets, m: int, device) -> Tensor:
    if isinstance(rows, Tensor):
        if rows.dtype != torch.int32 or rows.shape != (m,) or rows.device != device:
            raise ValueError(f"row indices: int32 [{m}] on {device}")
        return rows if rows.is_contiguous() else rows.contiguous()
    if len(rows) != m:
        raise ValueError(f"adapter_names: one name per row, {m} rows, got {len(rows)}")
    return sets[0].indices(rows)


def lora_linear4bit_group_multi(x: Tensor, bases, adapter_sets, rows: Union[Sequence[str], Tensor], x_loras=None):
    """`lora_linear4bit_group_mixed` for training: `[base_p(x) + per-row LoRA of adapter_sets[p]]` for 1..3 Linear4bit of one
    shape on one input, differentiable in `x`, in `x_loras` and in every adapter's lora_A and lora_B held by the sets, so one
    batch trains several adapters over one frozen base.  `rows`: the int32 row-index tensor of `LoraAdapterSet.indices`
    (an index outside [0, len(set)) means no adapter), or one name per row.  `x_loras`: each problem's dropped input (peft's
    `lora_dropout`), of x's shape; None: the adapters read x.  The sets hold the same names with the same ranks.

    Every token count takes the segmented path, so no host branch depends on the indices and a step can be captured in a
    CUDA graph or compiled.  The gradients of the adapters' weights are views of one flat buffer per problem and kind."""
    _refuse_dora(adapter_sets)
    cdt = _validate(x, bases, adapter_sets, training=True)
    if any(s.ranks != adapter_sets[0].ranks for s in adapter_sets):
        raise ValueError("grouped adapter sets must give each adapter the same rank")
    n = len(bases)
    if x_loras is not None:
        if len(x_loras) != n or any(t.shape != x.shape or t.device != x.device for t in x_loras):
            raise ValueError("x_loras: one input of x's shape per base")
    m = x.numel() // x.shape[-1] if x.shape[-1] else 0
    rows = _rows_tensor(rows, adapter_sets, m, x.device)
    tensors = [*(x_loras if x_loras is not None else [None] * n), *[b.weight.t() for b in bases], *[_bias(b, cdt) for b in bases],
               *[a for s in adapter_sets for a in s.lora_as], *[b for s in adapter_sets for b in s.lora_bs]]
    return MultiLoraMatMul4Bit.apply(x, rows, tuple(b.weight.quant_state for b in bases), tuple(adapter_sets), n, *tensors)


def lora_linear4bit_multi(x: Tensor, base, adapter_set: LoraAdapterSet, rows: Union[Sequence[str], Tensor],
                          x_lora: Tensor | None = None) -> Tensor:
    """`lora_linear4bit_group_multi` for one Linear4bit: `base(x)` plus each row's own adapter, trainable."""
    return lora_linear4bit_group_multi(x, [base], [adapter_set], rows, None if x_lora is None else [x_lora])[0]


# ----------------------------------------------------------------------------------------------------------------------
# training several DoRA adapters over one base in one batch (DESIGN.md §6e)
# ----------------------------------------------------------------------------------------------------------------------

class DoraAdapterSet(LoraAdapterSet):
    """The DoRA adapters of one linear, `{name: (lora_A.weight [r, K], lora_B.weight [N, r], magnitude [N], scaling)}` (peft's
    `use_dora=True`: the magnitude is `lora_magnitude_vector[name].weight`), built once.  `LoraAdapterSet`'s rules and
    device tables, plus a device table of the magnitudes' addresses (of the adapters' dtype, contiguous, 16-byte aligned) and
    the layouts of the stacked A rows and of the Gram matrices that the norms use.  The LoRA entry points refuse a
    DoraAdapterSet: they would drop its magnitudes."""

    def __init__(self, adapters: dict):
        if not adapters:
            raise ValueError("DoraAdapterSet: no adapters")
        for name, entry in adapters.items():
            if len(entry) != 4:
                raise ValueError(f"adapter {name!r}: (lora_A.weight, lora_B.weight, magnitude, scaling)")
        super().__init__({name: (a, b, s) for name, (a, b, _, s) in adapters.items()})
        self.magnitudes = []
        for name, (_, _, m, _) in adapters.items():
            if (m.dim() != 1 or m.shape[0] != self.out_features or m.dtype != self.dtype or m.device != self.device
                    or not m.is_contiguous() or m.data_ptr() % 16):
                raise ValueError(f"adapter {name!r}: a contiguous, 16-byte aligned {self.dtype} magnitude "
                                 f"[{self.out_features}] on {self.device}")
            self.magnitudes.append(m)
        self.mag_table = torch.tensor([m.data_ptr() for m in self.magnitudes], dtype=torch.int64).to(self.device)
        ranks = torch.tensor(self.ranks, dtype=torch.int64)
        # stacked row j of the norms' fused forward belongs to adapter stack_rows[j]; G_a sits at gram_offsets[a]
        self.stack_rows = torch.arange(len(self.ranks), dtype=torch.int32).repeat_interleave(ranks).to(self.device)
        sq = ranks * ranks
        self.gram_total = int(sq.sum())
        self.gram_offsets = (torch.cumsum(sq, 0) - sq).to(self.device)

    def requires_grad(self) -> bool:
        return super().requires_grad() or any(m.requires_grad for m in self.magnitudes)


def _refuse_dora(sets) -> None:
    if any(isinstance(s, DoraAdapterSet) for s in sets):
        raise ValueError("a DoraAdapterSet holds magnitudes that the LoRA entry points would drop: use "
                         "dora_linear4bit_group_multi / dora_linear4bit_multi")


class MultiDoraMatMul4Bit(torch.autograd.Function):
    """DoRA per row over n = 1..3 Linear4bit of one shape on one input (no bias): for row t with adapter a = rows[t] and
    c_{p,a} = m_{p,a} / ||W_p + s B_{p,a} A_{p,a}||_row (detached, fp32),
        no dropout  y_p[t] = c ⊙ (x[t] . W_p^T + U_p[t] . B_{p,a}^T)                       U_p[t] = rn(s . x[t] . A_{p,a}^T)
        dropout     y_p[t] = x[t] . W_p^T + (c - 1) ⊙ (xd_p[t] . W_p^T) + c ⊙ U_p[t] . B_{p,a}^T   U from xd_p
    and rows outside [0, n) take the base only.  Forward: the norms of every adapter (`dora_segmented_norm`), the base launch
    (and with dropout the grouped launch on the dropped inputs), then the segmented shrink and DoRA expand
    (`dora_segmented_fwd`).  Backward: `dora_grad_scale` (dQ, dD, dm), the base dX launches, then `dora_segmented_bwd`.
    Differentiable in x, the dropped inputs and every adapter's A, B and magnitude."""

    @staticmethod
    def forward(ctx, x, rows, states, sets, n: int, *tensors):
        x_loras, packeds = list(tensors[:n]), list(tensors[n:2 * n])
        cdt = sets[0].dtype
        x2d = F.as_compute_2d(x, cdt)
        split = x_loras[0] is not None
        xls = [F.as_compute_2d(t, cdt) for t in x_loras] if split else [x2d]
        states = list(states)
        n_ad, r = len(sets[0]), max(s.rmax for s in sets)
        n_out, k_in = states[0].shape
        sts = [F._state_tensors(qs, x2d.device) for qs in states]
        norm2s = [F.weight_row_norm2(p, qs) for p, qs in zip(packeds, states)]
        s0 = sets[0]
        cs, nrms = _ops.dora_segmented_norm([s.table for s in sets], [s.mag_table for s in sets], s0.stack_rows, s0.rank_offsets,
                                            s0.gram_offsets, s0.rank_total, s0.gram_total, packeds,
                                            [a_f32 if a_u8 is None else a_u8 for a_u8, _, _, _, a_f32 in sts],
                                            [t[1] for t in sts], [t[2] for t in sts], [t[3] for t in sts], n_out, k_in,
                                            states[0].dtype, norm2s, cdt, n_ad, r)
        outs = F.nf4_linear_group(False, [x2d] * n, packeds, states)
        qs = F.nf4_linear_group(False, xls, packeds, states) if split else []
        us, ws = _ops.dora_segmented_fwd(xls, [s.table for s in sets], rows, n_ad, r, cs, outs, qs)
        ctx.save_for_backward(us, ws, cs, nrms, *xls, *packeds, *(qs if split else outs))
        ctx.n, ctx.states, ctx.sets, ctx.r, ctx.split = n, states, sets, r, split
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.xl_meta = [(t.shape, t.dtype) for t in x_loras] if split else None
        out_dtype = F.out_dtype_for(x.dtype, cdt)
        return tuple((y if y.dtype == out_dtype else y.to(out_dtype)).view(*x.shape[:-1], n_out) for y in outs)

    @staticmethod
    def backward(ctx, *grad_ys):
        n, sets, split = ctx.n, ctx.sets, ctx.split
        us, ws, cs, nrms, *rest = ctx.saved_tensors
        n_xl = n if split else 1
        xls, packeds, qs = rest[:n_xl], rest[n_xl:n_xl + n], rest[n_xl + n:]
        need = ctx.needs_input_grad
        n_ad = len(sets[0])
        cdt = sets[0].dtype
        s0 = sets[0]
        tables = [s.table for s in sets]
        g2ds = [F.as_compute_2d(g, cdt) for g in grad_ys]
        dq, dd, dm = _ops.dora_grad_scale(g2ds, tables, s0.rank_offsets, s0.rank_total, list(qs), cs, nrms, ws, n_ad, ctx.r, split)
        if split:
            dx = F.nf4_linear_group(True, g2ds, packeds, ctx.states, out_dtype=cdt) if need[0] else None
            dxs = [F.nf4_linear_group(True, [dd[p]], [packeds[p]], [ctx.states[p]], out_dtype=cdt) for p in range(n)]
        else:
            dx = F.nf4_linear_group(True, list(dq.unbind(0)), packeds, ctx.states, out_dtype=cdt)
            dxs = [dx]
        d_a, d_b = _ops.dora_segmented_bwd(list(dq.unbind(0)), tables, s0.rank_offsets, s0.rank_total, us, list(xls), ws, n_ad,
                                           ctx.r, dxs)
        grad_x = None if dx is None or not need[0] else dx.to(ctx.x_dtype).view(ctx.x_shape)
        grad_xls = [None] * n
        if split:
            for p in range(n):
                if need[5 + p]:
                    shape, dtype = ctx.xl_meta[p]
                    grad_xls[p] = dxs[p].to(dtype).view(shape)
        k, n_out = xls[0].shape[1], g2ds[0].shape[1]
        offs, ranks = s0.rank_offsets_host, s0.ranks
        base = 5 + 2 * n
        grad_as = [d_a[p, offs[a] * k:(offs[a] + ranks[a]) * k].view(ranks[a], k) if need[base + p * n_ad + a] else None
                   for p in range(n) for a in range(n_ad)]
        base += n * n_ad
        grad_bs = [d_b[p, offs[a] * n_out:(offs[a] + ranks[a]) * n_out].view(n_out, ranks[a]) if need[base + p * n_ad + a] else None
                   for p in range(n) for a in range(n_ad)]
        base += n * n_ad
        grad_ms = [dm[p, a * n_out:(a + 1) * n_out] if need[base + p * n_ad + a] else None for p in range(n) for a in range(n_ad)]
        return (grad_x, None, None, None, None, *grad_xls, *([None] * n), *grad_as, *grad_bs, *grad_ms)


def dora_linear4bit_group_multi(x: Tensor, bases, dora_sets, rows: Union[Sequence[str], Tensor], x_loras=None):
    """`lora_linear4bit_group_multi` for DoRA: `[per-row DoRA of dora_sets[p] over base_p]` for 1..3 Linear4bit of one
    shape on one input (no bias), differentiable in `x`, in `x_loras` and in every adapter's lora_A, lora_B and magnitude
    held by the `DoraAdapterSet`s, so one batch trains several QDoRA adapters over one frozen base.  `rows` and `x_loras`
    as for `lora_linear4bit_group_multi`; the sets hold the same names with the same ranks.  Rows without an adapter
    return `Linear4bit`'s bits.  No host branch depends on the indices or on device values, so a step can be captured in a
    CUDA graph or compiled once the bases' row norms are cached (`functional.weight_row_norm2`).  The gradients of each
    kind (A, B, magnitude) are views of one flat buffer per problem."""
    if not all(isinstance(s, DoraAdapterSet) for s in dora_sets):
        raise ValueError("dora_linear4bit_group_multi: one DoraAdapterSet per base")
    cdt = _validate(x, bases, dora_sets, training=True)
    if any(s.ranks != dora_sets[0].ranks for s in dora_sets):
        raise ValueError("grouped adapter sets must give each adapter the same rank")
    if any(b.bias is not None for b in bases):
        raise ValueError("dora_linear4bit_group_multi: bases without bias")
    n = len(bases)
    if x_loras is not None:
        if len(x_loras) != n or any(t.shape != x.shape or t.device != x.device for t in x_loras):
            raise ValueError("x_loras: one input of x's shape per base")
    m = x.numel() // x.shape[-1] if x.shape[-1] else 0
    rows = _rows_tensor(rows, dora_sets, m, x.device)
    tensors = [*(x_loras if x_loras is not None else [None] * n), *[b.weight.t() for b in bases],
               *[a for s in dora_sets for a in s.lora_as], *[b for s in dora_sets for b in s.lora_bs],
               *[mg for s in dora_sets for mg in s.magnitudes]]
    return MultiDoraMatMul4Bit.apply(x, rows, tuple(b.weight.quant_state for b in bases), tuple(dora_sets), n, *tensors)


def dora_linear4bit_multi(x: Tensor, base, dora_set: DoraAdapterSet, rows: Union[Sequence[str], Tensor],
                          x_lora: Tensor | None = None) -> Tensor:
    """`dora_linear4bit_group_multi` for one Linear4bit: each row's own DoRA adapter over `base`, trainable."""
    return dora_linear4bit_group_multi(x, [base], [dora_set], rows, None if x_lora is None else [x_lora])[0]
