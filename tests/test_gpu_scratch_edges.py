"""The scratch path (each NF4 weight dequantized once per call into a bf16 scratch, then the TMA-fed GEMM of DESIGN.md 4.1) at
the edges that TMA zero-fill and tensor-map extents handle: partial feature blocks, contraction tails shorter than one
64-wide step, LoRA ranks that fill half of a k16 MMA step, fewer units than CTAs, and token counts of every residue of the
last token tile.  Checked against the C oracle's weights in float64, rounded to bf16 once.

Operands are also padded with bf16 NaN where a correct kernel never reads (a wrong extent turns NaN . 0 into a NaN output),
and calls are chained without host synchronization so that a misplaced programmatic-dependent-launch wait rewrites or reads
a recycled scratch while its neighbour launch still uses it.  Every case asserts that it takes the scratch path at the
library's natural threshold."""
import ctypes as ct

import numpy as np
import pytest
import torch

from gpu_helpers import assert_close_bf16, bf16_to_f32_np, make_act, make_weight, oracle_weight

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
TOL = 1e-3
RANKS = [8, 24, 40, 56]
# (M, N, K): forward last feature block 8 wide, dX contraction tail 8 of 64, dX last feature block 64 wide |
# forward last block 120 wide, dX tail 56 of 64, 86 feature blocks (full rounds plus a tail), T % 16 = 8 at 3000 |
# fewer units than CTAs, ragged in every dimension
SHAPES = [(2000, 4104, 4160), (2048, 11000, 1088), (3000, 11000, 1088), (1543, 200, 192)]


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    return F


def _lib():
    from qlora_b200 import _lib

    return _lib.load()


def _assert_scratch(m, n, k, nprob=1, is_bwd=False):
    assert _lib().qb200_nf4_linear_scratch_size(nprob, m, n, k, int(is_bwd)) == nprob * n * k * 2


def _quant(F, n, k, seed, nested=True, state_dtype=BF16):
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=seed, dtype=state_dtype), compress_statistics=nested, quant_type="nf4")
    assert qs.dtype == state_dtype
    return packed.t(), qs


def _w64(F, packed, qs, c_oracle):
    """The oracle's bf16 weight [N, K] as float64 on the GPU."""
    return torch.from_numpy(oracle_weight(packed, qs, c_oracle)).cuda().double()


def _check(y, ref64):
    """The parity bar against a float64 reference rounded to bf16 once."""
    assert y.dtype == BF16
    assert_close_bf16(bf16_to_f32_np(y), ref64.float().to(BF16).float().cpu().numpy(), TOL)


def _nan_buffer(rows, cols):
    return torch.full((rows, cols), float("nan"), dtype=BF16, device="cuda")


def _padded(t, extra_rows=256, extra_cols=64):
    """`t` [R, C] as the top-left view of an [R + extra_rows, C + extra_cols] buffer that is NaN elsewhere."""
    buf = _nan_buffer(t.shape[0] + extra_rows, t.shape[1] + extra_cols)
    buf[:t.shape[0], :t.shape[1]] = t
    return buf[:t.shape[0], :t.shape[1]]


def _slices(ts, extra_rows=256, extra_cols=64):
    """Equal-width [T, r] tensors as column slices, side by side, of one [T + extra_rows, nprob r + extra_cols] buffer that is
    NaN outside them."""
    t, r = ts[0].shape
    buf = _nan_buffer(t + extra_rows, len(ts) * r + extra_cols)
    for i, x in enumerate(ts):
        buf[:t, i * r:(i + 1) * r] = x
    return [buf[:t, i * r:(i + 1) * r] for i in range(len(ts))]


def _direct(F, is_bwd, xs, ps, qss, ws, us=None, vs=None, out_dtype=BF16):
    """`qb200_nf4_linear_group_ex` called with the caller's workspace `ws` (a uint8 tensor) as the weight scratch."""
    from qlora_b200._lib import DTYPE_CODE, Nf4Problem

    lib = _lib()
    n_out, k_in = qss[0].shape
    m = xs[0].shape[0]
    outs = [torch.empty((m, k_in if is_bwd else n_out), dtype=out_dtype, device="cuda") for _ in range(1 if is_bwd else len(ps))]
    probs = (Nf4Problem * len(ps))()
    for i, (x, p, qs) in enumerate(zip(xs, ps, qss)):
        assert x.stride(1) == 1 and p.is_contiguous()
        a_u8, code, a2, off, a32 = F._state_tensors(qs, x.device)
        pr = probs[i]
        pr.inp, pr.ld_in, pr.packed = x.data_ptr(), x.stride(0), p.data_ptr()
        pr.absmax_u8, pr.code256, pr.absmax2, pr.offset, pr.absmax_f32 = (None if t is None else t.data_ptr()
                                                                          for t in (a_u8, code, a2, off, a32))
        if us is not None:
            assert vs[i].is_contiguous()
            pr.U, pr.ld_u, pr.V = us[i].data_ptr(), us[i].stride(0), vs[i].data_ptr()
        if i < len(outs):
            pr.out, pr.ld_out = outs[i].data_ptr(), outs[i].stride(0)
    r = 0 if us is None else us[0].shape[1]
    rc = lib.qb200_nf4_linear_group_ex(int(is_bwd), DTYPE_CODE[BF16], DTYPE_CODE[qss[0].dtype], len(ps), ct.addressof(probs), r, m,
                                       n_out, k_in, DTYPE_CODE[out_dtype], ws.data_ptr(), ws.numel(), F.stream_ptr(xs[0].device))
    assert rc == 0, lib.qb200_last_error()
    return outs[0] if is_bwd else outs


# ---- 1. parity with the oracle at ragged shapes ------------------------------------------------------------------------

STATES = [(s, True, BF16) for s in SHAPES] + [(s, False, BF16) for s in SHAPES] + [(SHAPES[2], True, F32)]
STATE_IDS = ["x".join(map(str, s)) + ("-nested" if nested else "-plain") + ("-f32state" if dt == F32 else "") for s, nested, dt in STATES]


@pytest.mark.parametrize("shape,nested,state_dtype", STATES, ids=STATE_IDS)
def test_scratch_matches_oracle_at_ragged_shapes(F, c_oracle, shape, nested, state_dtype):
    """Forward with bias, with LoRA and bias at every rank, with an fp32 output; dX, with LoRA at every rank, with an fp32
    output."""
    m, n, k = shape
    _assert_scratch(m, n, k)
    _assert_scratch(m, n, k, is_bwd=True)
    packed, qs = _quant(F, n, k, seed=n + k + m, nested=nested, state_dtype=state_dtype)
    w = _w64(F, packed, qs, c_oracle)
    x, dy = make_act(m, k, seed=1), make_act(m, n, seed=2)
    bias = make_weight(1, n, seed=3, scale=0.5).view(-1)

    base = x.double() @ w.t() + bias.double()
    y = F.nf4_linear_fwd(x, packed, qs, bias)
    _check(y, base)
    y32 = F.nf4_linear_fwd(x, packed, qs, bias, out_dtype=F32)
    assert y32.dtype == F32 and torch.equal(y32, y.float())
    for r in RANKS:
        u, v = make_act(m, r, seed=10 + r), make_weight(n, r, seed=20 + r, scale=0.05)
        _check(F.nf4_linear_fwd_lora(x, packed, qs, u, v, bias), base + u.double() @ v.double().t())
    del base

    base = dy.double() @ w
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    _check(dx, base)
    dx32 = F.nf4_linear_bwd_dx(dy, packed, qs, out_dtype=F32)
    assert dx32.dtype == F32 and torch.equal(dx32, dx.float())
    for r in RANKS:
        g, a = make_act(m, r, seed=30 + r), make_weight(r, k, seed=40 + r, scale=0.05)
        _check(F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a), base + g.double() @ a.double())


@pytest.mark.parametrize("nprob,m,n,k", [(3, 2000, 4104, 4160), (2, 2048, 11000, 1088)], ids=["qkv", "gate_up"])
def test_scratch_grouped_matches_oracle_at_ragged_shapes(F, c_oracle, nprob, m, n, k):
    """q/k/v and gate/up with LoRA at every rank: U (and G) are column slices of one [T, nprob r] buffer, the forward outputs
    column slices of one [T, nprob N] buffer, and dX sums the problems in one output."""
    _assert_scratch(m, n, k, nprob)
    _assert_scratch(m, n, k, nprob, is_bwd=True)
    ps, qss = zip(*[_quant(F, n, k, seed=17 * i + n) for i in range(nprob)])
    ws = [_w64(F, p, qs, c_oracle) for p, qs in zip(ps, qss)]
    x = make_act(m, k, seed=1)
    dys = [make_act(m, n, seed=2 + i) for i in range(nprob)]
    fwd = [x.double() @ w.t() for w in ws]
    bwd = sum(dy.double() @ w for dy, w in zip(dys, ws))
    for r in RANKS:
        ubuf = torch.cat([make_act(m, r, seed=100 * r + i) for i in range(nprob)], dim=1)
        us = [ubuf[:, i * r:(i + 1) * r] for i in range(nprob)]
        vs = [make_weight(n, r, seed=200 * r + i, scale=0.05) for i in range(nprob)]
        ybuf = torch.empty((m, nprob * n), dtype=BF16, device="cuda")
        ys = F.nf4_linear_group(False, [x] * nprob, list(ps), list(qss), us=us, vs=vs,
                                outs=[ybuf[:, i * n:(i + 1) * n] for i in range(nprob)])
        for i, y in enumerate(ys):
            assert y.data_ptr() == ybuf[:, i * n:].data_ptr()
            _check(y, fwd[i] + us[i].double() @ vs[i].double().t())
        gbuf = torch.cat([make_act(m, r, seed=300 * r + i) for i in range(nprob)], dim=1)
        gs = [gbuf[:, i * r:(i + 1) * r] for i in range(nprob)]
        as_ = [make_weight(r, k, seed=400 * r + i, scale=0.05) for i in range(nprob)]
        dx = F.nf4_linear_group(True, dys, list(ps), list(qss), us=gs, vs=as_)
        _check(dx, bwd + sum(g.double() @ a.double() for g, a in zip(gs, as_)))


def test_scratch_token_count_sweep(F, c_oracle):
    """Forward with LoRA at T = 1536 + 16 j and 1543 + 16 j, j = 0..16: the last token tile of each feature block takes every
    multiple of 16 (and every multiple of 16 plus 7) below 256, with the rank cycling through 8, 24, 40, 56."""
    n, k = 11000, 1088
    ts = [1536 + 16 * j for j in range(17)] + [1543 + 16 * j for j in range(17)]
    packed, qs = _quant(F, n, k, seed=5)
    w = _w64(F, packed, qs, c_oracle)
    x = make_act(max(ts), k, seed=6)
    base = x.double() @ w.t()
    for j, t in enumerate(ts):
        _assert_scratch(t, n, k)
        r = RANKS[j % len(RANKS)]
        u, v = make_act(t, r, seed=7 + j), make_weight(n, r, seed=8 + j, scale=0.05)
        _check(F.nf4_linear_fwd_lora(x[:t], packed, qs, u, v), base[:t] + u.double() @ v.double().t())


# ---- 2. reads stay inside each operand ---------------------------------------------------------------------------------

@pytest.mark.parametrize("nprob,m,n,k", [(3, 2000, 4104, 4160), (2, 3000, 11000, 1088)], ids=["qkv", "gate_up"])
@pytest.mark.parametrize("padded", ["activations", "lora", "scratch"])
def test_reads_stay_inside_each_operand(F, nprob, m, n, k, padded):
    """Single and grouped, forward and dX, with LoRA (r = 24), NaN placed where a correct kernel never reads:
    activations: X and dY as [T, C] views of [T + 256, C + 64] buffers (dX reads a contraction tail of N % 64 columns);
    lora: U / G as column slices of a [T + 256, nprob r + 64] buffer, and the dX LoRA A [r, K] as the first r rows of an
          [r + 64, K] buffer;
    scratch: the weight scratch lent to qb200_nf4_linear_group_ex exactly as large as the call needs plus 64 K bf16 values,
          all bytes 0xFF before the call (the dX weight map must end at row N).
    Every output is finite and bitwise equal to the same call with unpadded operands."""
    r = 24
    _assert_scratch(m, n, k, nprob)
    _assert_scratch(m, n, k, nprob, is_bwd=True)
    ps, qss = zip(*[_quant(F, n, k, seed=23 * i + k) for i in range(nprob)])
    ps = [p.contiguous() for p in ps]
    x = make_act(m, k, seed=1)
    dys = [make_act(m, n, seed=2 + i) for i in range(nprob)]
    us = [make_act(m, r, seed=10 + i) for i in range(nprob)]
    vs = [make_weight(n, r, seed=20 + i, scale=0.05) for i in range(nprob)]
    gs = [make_act(m, r, seed=30 + i) for i in range(nprob)]
    as_ = [make_weight(r, k, seed=40 + i, scale=0.05) for i in range(nprob)]
    px, pdys, pus, pgs, pas = x, dys, us, gs, as_
    if padded == "activations":
        px, pdys = _padded(x), [_padded(dy) for dy in dys]
    elif padded == "lora":
        pus, pgs = _slices(us), _slices(gs)
        pas = [_padded(a, extra_rows=64, extra_cols=0) for a in as_]
    assert all(p.is_contiguous() for p in pas)

    # the unpadded calls get the same room after the scratch, zeroed
    ws_bytes = nprob * n * k * 2 + 64 * k * 2
    clean = torch.zeros(ws_bytes, dtype=torch.uint8, device="cuda")

    def workspace():
        if padded != "scratch":
            return clean
        return torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")

    for p in (1, nprob):
        ref_f = _direct(F, False, [x] * p, ps[:p], qss[:p], clean, us[:p], vs[:p])
        got_f = _direct(F, False, [px] * p, ps[:p], qss[:p], workspace(), pus[:p], vs[:p])
        ref_b = _direct(F, True, dys[:p], ps[:p], qss[:p], clean, gs[:p], as_[:p])
        got_b = _direct(F, True, pdys[:p], ps[:p], qss[:p], workspace(), pgs[:p], pas[:p])
        torch.cuda.synchronize()
        for got, ref in zip(got_f + [got_b], ref_f + [ref_b]):
            assert bool(torch.isfinite(got).all()) and torch.equal(got, ref)


# ---- 4. ordering across calls ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nested", [True, False])
def test_scratch_calls_right_after_quantize(F, nested):
    """The scratch path's dequantize is a programmatic dependent launch that loads the quant state before it waits for the
    previous kernel.  Quantize, then a forward and a dX of the fresh weight with no sync in between, for three weights: each
    result bitwise that of the same call after a sync."""
    m, n, k = 2048, 4104, 4160
    _assert_scratch(m, n, k)
    _assert_scratch(m, n, k, is_bwd=True)
    x, dy = make_act(m, k, seed=1), make_act(m, n, seed=2)
    weights = [make_weight(n, k, seed=60 + i) for i in range(3)]
    torch.cuda.synchronize()
    got = []
    for w in weights:
        packed, qs = F.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
        got.append((packed, qs, F.nf4_linear_fwd(x, packed.t(), qs), F.nf4_linear_bwd_dx(dy, packed.t(), qs)))
    for packed, qs, y, dx in got:
        torch.cuda.synchronize()
        ry = F.nf4_linear_fwd(x, packed.t(), qs)
        torch.cuda.synchronize()
        rdx = F.nf4_linear_bwd_dx(dy, packed.t(), qs)
        torch.cuda.synchronize()
        assert torch.equal(y, ry) and torch.equal(dx, rdx)


def test_scratch_chain_reads_the_previous_output(F):
    """Forward, forward, dX on a square W, each call's input the previous call's output, no sync in between: bitwise the
    same calls with a sync around each."""
    m, n = 2048, 2112
    _assert_scratch(m, n, n)
    packed, qs = _quant(F, n, n, seed=80)
    x = make_act(m, n, seed=81)
    torch.cuda.synchronize()
    y1 = F.nf4_linear_fwd(x, packed, qs)
    y2 = F.nf4_linear_fwd(y1, packed, qs)
    d = F.nf4_linear_bwd_dx(y2, packed, qs)
    refs = []
    inp = x
    for fn in (F.nf4_linear_fwd, F.nf4_linear_fwd, F.nf4_linear_bwd_dx):
        torch.cuda.synchronize()
        inp = fn(inp, packed, qs)
        torch.cuda.synchronize()
        refs.append(inp)
    for got, ref in zip((y1, y2, d), refs):
        assert torch.equal(got, ref)


def _two_weight_sequence(F, ws=None):
    """W1 forward, W2 forward, W1 dX, W2 dX, then the grouped dX of both, with no sync: through one workspace `ws` lent to
    the C entry point, or (ws None) through `functional`, whose per-call scratch the caching allocator hands on."""
    m, n, k = 2048, 4104, 4160
    ps, qss = zip(*[_quant(F, n, k, seed=90 + i) for i in range(2)])
    ps = [p.contiguous() for p in ps]
    x = make_act(m, k, seed=91)
    dys = [make_act(m, n, seed=92 + i) for i in range(2)]
    calls = [(False, [x], [0]), (False, [x], [1]), (True, dys[:1], [0]), (True, dys[1:], [1]), (True, dys, [0, 1])]

    def run(i):
        is_bwd, xs, idx = calls[i]
        pp, qq = [ps[j] for j in idx], [qss[j] for j in idx]
        if ws is not None:
            out = _direct(F, is_bwd, xs, pp, qq, ws)
        else:
            out = F.nf4_linear_group(is_bwd, xs, pp, qq)
        return out if is_bwd else out[0]

    return len(calls), run


@pytest.mark.parametrize("entry", ["functional", "workspace"])
def test_different_weights_through_one_recycled_scratch(F, entry):
    """Each output of the unsynchronized sequence is bitwise that call run alone after a sync: a dequantize that stored
    before the previous GEMM stopped reading the scratch, or a GEMM that loaded before its dequantize finished, would mix
    the two weights."""
    m, n, k = 2048, 4104, 4160
    _assert_scratch(m, n, k, 2, is_bwd=True)
    ws = torch.empty(2 * n * k * 2, dtype=torch.uint8, device="cuda") if entry == "workspace" else None
    ncalls, run = _two_weight_sequence(F, ws)
    torch.cuda.synchronize()
    got = [run(i) for i in range(ncalls)]
    for i in range(ncalls):
        torch.cuda.synchronize()
        ref = run(i)
        torch.cuda.synchronize()
        assert torch.equal(got[i], ref), i


@pytest.mark.parametrize("entry", ["functional", "workspace"])
def test_recycled_scratch_sequence_replays_under_cuda_graphs(F, entry):
    """The same sequence captured in one CUDA graph (as the bench replays its step) and replayed once."""
    ws = torch.empty(2 * 4104 * 4160 * 2, dtype=torch.uint8, device="cuda") if entry == "workspace" else None
    ncalls, run = _two_weight_sequence(F, ws)
    torch.cuda.synchronize()
    eager = []
    for i in range(ncalls):
        eager.append(run(i))
        torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(ncalls):   # warm-up: tensor maps, kernel attributes, schedules
            run(i)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = [run(i) for i in range(ncalls)]
    for t in static:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(static, eager)):
        assert torch.equal(a, b), i
