"""GPU parity of bf16 compute over fp16 and fp32 quant states, and of the fp16 output under bf16 compute.

`BitsAndBytesConfig(..., bnb_4bit_compute_dtype=torch.bfloat16)` over an fp16 checkpoint quantizes fp16 weights (fp16 state)
and feeds fp16 activations; over a model loaded in fp32 the state is fp32.  The reference for the fused kernels is this
library's unfused path `dequantize_4bit(W, state).to(bf16)`:
    fp32 state: bf16_rn(LUT[j] * absmax)                 fp16 state: bf16_rn(fp16_rn(LUT[j] * absmax))  (two roundings)
and an fp16 output is the bf16-rounded result rounded to fp16, what `Linear4bit.forward`'s `.to(fp16)` gives.
Parity bar: DESIGN.md §2 (bf16): Frobenius-relative error <= 1e-3 and every element within one bf16 ulp of max|ref|."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fp16_helpers import f16_round, np32, oracle_w32
from gpu_helpers import assert_close_bf16, make_act, make_weight, rel_err
from oracle import nf4_oracle as o

pytestmark = pytest.mark.gpu
BF, H16, F32 = torch.bfloat16, torch.float16, torch.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def q():
    import qlora_b200 as q

    assert torch.cuda.is_available() and q._lib.load().qb200_has_fused_gemm() == 1
    return q


def quantized(q, n, k, seed, state_dtype, nested=True, tiny_rows=0):
    """NF4 state of an [n, k] weight of `state_dtype`; the first `tiny_rows` rows are scaled by 1e-3 so that their blocks'
    products fall below fp16's smallest normal (6.1e-5): fp16 subnormals."""
    w = make_weight(n, k, seed, dtype=F32)
    if tiny_rows:
        w[:tiny_rows] *= 1e-3
    packed, qs = q.functional.quantize_4bit(w.to(state_dtype), compress_statistics=nested, quant_type="nf4")
    assert qs.dtype == state_dtype
    return packed, qs


def ref_weight(c_oracle, packed, qs):
    """The weight `dequantize_4bit(W, state).to(bf16)` returns, from the C oracle's fp32 products rounded by numpy."""
    w32 = oracle_w32(c_oracle, packed, qs)
    return o.bf16_round(f16_round(w32) if qs.dtype == H16 else w32)


def bf16_bits(t):
    return t.detach().view(torch.int16).cpu().numpy()


def np_bits(a):
    return (np.asarray(a, np.float32).view(np.uint32) >> 16).astype(np.uint16).view(np.int16)


def act(m, k, seed, scale=1.0, dtype=BF):
    return (make_act(m, k, seed).float() * scale).to(dtype)


def gpu_ref(a, w, extra=None):
    """fp64 GEMM on the GPU of fp32 operands (exact products, one rounding left to the caller)."""
    r = torch.as_tensor(a, device="cuda").double() @ torch.as_tensor(w, device="cuda").double()
    if extra is not None:
        r = r + torch.as_tensor(extra, device="cuda").double()
    return r.float().cpu().numpy()


# ---------------------------------------------------------------- exact weights -------------------------------------------

@pytest.mark.parametrize("state_dtype", [H16, F32])
@pytest.mark.parametrize("nested", [True, False])
def test_identity_reads_double_rounded_weights(q, c_oracle, nested, state_dtype):
    """Identity GEMMs (K-major forward, MN-major dX) and one-hot skinny calls return the weights bit for bit: the oracle's
    fp32 products rounded by numpy, twice for an fp16 state; equal to `dequantize_4bit(...).to(bf16)` too.  The fp16 output
    of the same launches is those weights rounded to fp16."""
    F = q.functional
    n, k = 384, 320
    packed, qs = quantized(q, n, k, seed=11, state_dtype=state_dtype, nested=nested, tiny_rows=32)
    w = ref_weight(c_oracle, packed, qs)
    if state_dtype == H16:
        w32 = oracle_w32(c_oracle, packed, qs)
        f16 = f16_round(w32)
        assert (np.abs(f16[:32]) < 2.0 ** -14).any() and (f16[:32] != 0).any()          # fp16 subnormals occur
        assert (w != o.bf16_round(w32)).sum() > 0                                         # two roundings differ from one
    assert np.array_equal(bf16_bits(F.dequantize_4bit(packed, qs).to(BF)), np_bits(w))
    y = F.nf4_linear_fwd(torch.eye(k, dtype=BF, device="cuda"), packed, qs)
    assert y.dtype == BF and np.array_equal(bf16_bits(y), np_bits(np.ascontiguousarray(w.T)))
    dx = F.nf4_linear_bwd_dx(torch.eye(n, dtype=BF, device="cuda"), packed, qs)
    assert np.array_equal(bf16_bits(dx), np_bits(w))
    assert torch.equal(F.nf4_linear_fwd(torch.eye(k, dtype=BF, device="cuda"), packed, qs, out_dtype=H16), y.to(H16))
    assert torch.equal(F.nf4_linear_bwd_dx(torch.eye(n, dtype=BF, device="cuda"), packed, qs, out_dtype=H16), dx.to(H16))
    # skinny kernels: token t of a one-hot batch selects column cols[t] of W
    for m in (1, 8, 16):
        cols = [(37 * t + 5) % k for t in range(m)]
        x = torch.zeros(m, k, dtype=BF, device="cuda")
        x[torch.arange(m), torch.tensor(cols)] = 1
        ys = F.nf4_linear_fwd(x, packed, qs)
        assert np.array_equal(bf16_bits(ys), np_bits(np.ascontiguousarray(w[:, cols].T)))
        assert torch.equal(F.nf4_linear_fwd(x, packed, qs, out_dtype=H16), ys.to(H16))


# ---------------------------------------------------------------- parity --------------------------------------------------

SMALL = (384, 320)
MODEL_SHAPES = [(4096, 4096), (11008, 4096), (4096, 11008)]     # Llama-2-7B: q/k/v/o, gate/up, down
TOKENS = [1, 7, 16, 17, 100, 300, 2048]


def _check_fwd_dx(q, c_oracle, m, n, k, state_dtype, seed):
    F = q.functional
    packed, qs = quantized(q, n, k, seed=seed, state_dtype=state_dtype)
    w = ref_weight(c_oracle, packed, qs)
    x, dy = act(m, k, 1), act(m, n, 2)
    bias = make_weight(1, n, seed=3, scale=0.5).view(-1)
    y = F.nf4_linear_fwd(x, packed, qs, bias)
    assert_close_bf16(np32(y), o.bf16_round(gpu_ref(np32(x), w.T, np32(bias))))
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    assert_close_bf16(np32(dx), o.bf16_round(gpu_ref(np32(dy), w)))
    # the fold: fp16 output == bf16 output cast to fp16; fp32 output == bf16 output widened
    assert torch.equal(F.nf4_linear_fwd(x, packed, qs, bias, out_dtype=H16), y.to(H16))
    assert torch.equal(F.nf4_linear_bwd_dx(dy, packed, qs, out_dtype=H16), dx.to(H16))
    if m > 16:   # an fp32 output never takes the skinny kernels
        assert torch.equal(F.nf4_linear_fwd(x, packed, qs, bias, out_dtype=F32), y.float())


@pytest.mark.parametrize("m", TOKENS)
@pytest.mark.parametrize("n,k", [SMALL] + MODEL_SHAPES)
def test_fp16_state_vs_oracle(q, c_oracle, m, n, k):
    """Forward (skinny kernels up to 16 tokens, split-K where the library plans it, the range schedule above) and dX."""
    _check_fwd_dx(q, c_oracle, m, n, k, H16, seed=n * 7 + k + m)


@pytest.mark.parametrize("m", TOKENS)
def test_fp32_state_vs_oracle(q, c_oracle, m):
    _check_fwd_dx(q, c_oracle, m, *SMALL, F32, seed=m)


@pytest.mark.parametrize("m", [17, 48, 300])
def test_split_k_with_lora_and_fold(q, c_oracle, m):
    """Split-K (fp32 partials + reduce) with LoRA operands over an fp16 state; the reduce's fp16 output equals its bf16 output
    cast to fp16."""
    F = q.functional
    lib = q._lib.load()
    n, k, r = 2048, 4096, 64
    if m <= 48:
        assert lib.qb200_nf4_linear_workspace_size(m, n, k, 0) > 0 and lib.qb200_nf4_linear_workspace_size(m, n, k, 1) > 0
    packed, qs = quantized(q, n, k, seed=77, state_dtype=H16)
    w = ref_weight(c_oracle, packed, qs)
    x, dy = act(m, k, 1), act(m, n, 2)
    u, v, a = act(m, r, 4, 0.5), make_weight(n, r, 5, scale=0.2), make_weight(r, k, 6, scale=0.2)
    y = F.nf4_linear_fwd_lora(x, packed, qs, u, v)
    assert_close_bf16(np32(y), o.bf16_round(gpu_ref(np32(x), w.T, np32(u) @ np32(v).T)))
    dx = F.nf4_linear_bwd_dx_lora(dy, packed, qs, u, a)
    assert_close_bf16(np32(dx), o.bf16_round(gpu_ref(np32(dy), w, np32(u) @ np32(a))))
    assert torch.equal(F.nf4_linear_fwd_lora(x, packed, qs, u, v, out_dtype=H16), y.to(H16))
    assert torch.equal(F.nf4_linear_bwd_dx_lora(dy, packed, qs, u, a, out_dtype=H16), dx.to(H16))


@pytest.mark.parametrize("state_dtype", [H16, F32])
@pytest.mark.parametrize("m,n,k,r,nprob", [(300, 200, 192, 16, 3), (7, 384, 320, 16, 3), (2048, 512, 1024, 64, 2), (1, 256, 128, 8, 2)])
def test_grouped_launches_with_lora_bias_and_fold(q, c_oracle, m, n, k, r, nprob, state_dtype):
    """q/k/v (3) and gate/up (2) as one launch per direction over fp16 / fp32 states, with LoRA operands and bias; the fp16
    outputs equal the bf16 outputs cast to fp16."""
    F = q.functional
    packs, states, ws = [], [], []
    for i in range(nprob):
        packed, qs = quantized(q, n, k, seed=31 * i + n + k, state_dtype=state_dtype)
        packs.append(packed)
        states.append(qs)
        ws.append(ref_weight(c_oracle, packed, qs))
    x = act(m, k, 1)
    biases = [make_weight(1, n, seed=60 + i, scale=0.5).view(-1) for i in range(nprob)]
    u_cat = act(m, nprob * r, 2, 0.5)
    us = [u_cat[:, i * r:(i + 1) * r] for i in range(nprob)]
    vs = [make_weight(n, r, 20 + i, scale=0.2) for i in range(nprob)]
    gs = [act(m, r, 40 + i, 0.5) for i in range(nprob)]
    as_ = [make_weight(r, k, 50 + i, scale=0.2) for i in range(nprob)]
    ys = F.nf4_linear_group(False, [x] * nprob, packs, states, biases, us=us, vs=vs)
    for i in range(nprob):
        ref = gpu_ref(np32(x), ws[i].T, np32(us[i]) @ np32(vs[i]).T + np32(biases[i]))
        assert_close_bf16(np32(ys[i]), o.bf16_round(ref))
    ys16 = F.nf4_linear_group(False, [x] * nprob, packs, states, biases, us=us, vs=vs, out_dtype=H16)
    assert all(torch.equal(a_, b_.to(H16)) for a_, b_ in zip(ys16, ys))
    dys = [act(m, n, 30 + i) for i in range(nprob)]
    dx = F.nf4_linear_group(True, dys, packs, states, us=gs, vs=as_)
    acc = sum(gpu_ref(np32(dys[i]), ws[i], np32(gs[i]) @ np32(as_[i])) for i in range(nprob))
    assert_close_bf16(np32(dx), o.bf16_round(acc))
    assert torch.equal(F.nf4_linear_group(True, dys, packs, states, us=gs, vs=as_, out_dtype=H16), dx.to(H16))


def test_group_needs_one_weight_rounding(q):
    """An fp16 state and a bf16 state in one bf16 launch would need two product tables: refused."""
    F = q.functional
    p1, s1 = quantized(q, 128, 128, seed=1, state_dtype=H16)
    p2, s2 = quantized(q, 128, 128, seed=2, state_dtype=BF)
    with pytest.raises(AssertionError, match="rounding"):
        F.nf4_linear_group(False, [act(4, 128, 1)] * 2, [p1, p2], [s1, s2])


# ---------------------------------------------------------------- module, autograd, graphs ---------------------------------

def _linear(q, n_in, n_out, state_dtype, bias=True, seed=0):
    torch.manual_seed(seed)
    lin = q.nn.Linear4bit(n_in, n_out, bias=bias, compute_dtype=BF, compress_statistics=True, quant_type="nf4")
    lin.weight.data = lin.weight.data.to(state_dtype)
    if bias:
        lin.bias.data = torch.randn(n_out) * 0.1
    lin = lin.cuda()
    assert lin.weight.quant_state.dtype == state_dtype
    return lin


@pytest.mark.parametrize("x_dtype,state_dtype", [(H16, H16), (H16, BF), (F32, F32)])
def test_module_folds_the_casts(q, x_dtype, state_dtype):
    """Linear4bit(compute_dtype=bf16): fp16 input over an fp16 or bf16 state, fp32 input over an fp32 state.  One fused launch
    per direction, the output and x.grad of the input's dtype, equal to the explicit cast -> fused -> cast sequence."""
    F = q.functional
    lin = _linear(q, 512, 768, state_dtype)
    qs, packed = lin.weight.quant_state, lin.weight.data
    x = torch.randn(3, 40, 512, device="cuda").to(x_dtype).requires_grad_(True)
    gy = torch.randn(3, 40, 768, device="cuda").to(x_dtype)
    n0 = F.LAUNCH_COUNTER[0]
    y = lin(x)
    y.backward(gy)
    assert F.LAUNCH_COUNTER[0] - n0 == 2
    assert y.dtype == x_dtype and x.grad.dtype == x_dtype
    y_ref = F.nf4_linear_fwd(x.detach().to(BF).view(-1, 512), packed, qs, lin.bias.detach().to(BF)).to(x_dtype)
    dx_ref = F.nf4_linear_bwd_dx(gy.to(BF).view(-1, 768), packed, qs).to(x_dtype)
    assert torch.equal(y.detach().view(-1, 768), y_ref) and torch.equal(x.grad.view(-1, 512), dx_ref)


def test_module_vs_unfused_path(q, c_oracle):
    """The fused fp16-state module against today's unfused path (USE_FUSED = False) and the oracle: same weights, so the
    results differ only by summation order."""
    lin = _linear(q, 512, 768, H16)
    w = ref_weight(c_oracle, lin.weight.data, lin.weight.quant_state)
    x = torch.randn(100, 512, device="cuda").to(H16)
    y = lin(x)
    q.autograd.USE_FUSED = False
    try:
        y_unf = lin(x)
    finally:
        q.autograd.USE_FUSED = True
    ref = o.bf16_round(gpu_ref(np32(x.to(BF)), w.T, np32(lin.bias.to(BF))))
    assert_close_bf16(np32(y), ref)
    assert_close_bf16(np32(y_unf), ref)


def test_module_cuda_graph_replay_equals_eager(q):
    lin = _linear(q, 512, 1024, H16, bias=True)
    x_static = torch.randn(700, 512, device="cuda", dtype=H16).requires_grad_(True)
    gy = torch.randn(700, 1024, device="cuda", dtype=H16)

    def fwd_bwd():
        x_static.grad = None
        y = lin(x_static)
        y.backward(gy)
        return y.detach(), x_static.grad

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = fwd_bwd()
    for seed in (1, 2):
        with torch.no_grad():
            x_static.copy_(torch.randn(700, 512, generator=torch.Generator().manual_seed(seed)).to(H16))
        g.replay()
        got = [t.clone() for t in outs]
        ref = [t.clone() for t in fwd_bwd()]
        assert all(torch.equal(a_, b_) for a_, b_ in zip(got, ref))


@pytest.mark.parametrize("m", [1, 4, 16])
def test_folded_skinny_pdl_chain(q, m):
    """A decode chain of grouped folded skinny launches (fp16 state, fp16 output; one launch per problem, chained by
    programmatic dependent launch), each step reading the previous step's output, equals the same launches with a
    synchronize between them."""
    F = q.functional
    n = k = 2048
    x0 = act(m, k, 70, 0.5)
    for it in range(3):
        pq = [quantized(q, n, k, seed=100 + 3 * it + i, state_dtype=H16) for i in range(3)]
        packs, states = [p for p, _ in pq], [s for _, s in pq]

        def step(x):
            return F.nf4_linear_group(False, [x] * 3, packs, states, out_dtype=H16)

        ys1 = step(x0)
        ys2 = step(ys1[2].to(BF))
        torch.cuda.synchronize()
        r1 = step(x0)
        torch.cuda.synchronize()
        r2 = step(r1[2].to(BF))
        torch.cuda.synchronize()
        assert all(a_.dtype == H16 and torch.equal(a_, b_) for a_, b_ in zip(ys1 + ys2, r1 + r2))


# ---------------------------------------------------------------- LoRA and DoRA ---------------------------------------------

def _adapters(n_in, n_out, r, count, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    As = [(torch.randn(r, n_in, generator=g) * 0.05).to(BF).cuda().requires_grad_(True) for _ in range(count)]
    Bs = [(torch.randn(n_out, r, generator=g) * 0.05).to(BF).cuda().requires_grad_(True) for _ in range(count)]
    return As, Bs


def _unfused(q, fn):
    q.autograd.USE_FUSED = False
    try:
        return fn()
    finally:
        q.autograd.USE_FUSED = True


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("m", [4, 300])
def test_lora_linear4bit_matches_unfused(q, dropout, m):
    """`lora_linear4bit` over an fp16 state with bf16 adapters and x, fused, against the unfused two-step form."""
    F = q.functional
    base = _linear(q, 512, 768, H16, bias=False)
    (A,), (B,) = _adapters(512, 768, 64, 1, seed=1)
    x = act(m, 512, 3).view(1, m, 512).requires_grad_(True)
    gy = act(m, 768, 4).view(1, m, 768)
    mask = ((torch.rand(1, m, 512, device="cuda") >= 0.1).float() / 0.9).to(BF)
    assert q.lora._group_fusable(x, [base], [A], [B], None)
    n0 = F.LAUNCH_COUNTER[0]
    y = q.lora_linear4bit(x, base, A, B, 0.25, x_lora=x * mask if dropout else None)
    assert F.LAUNCH_COUNTER[0] - n0 == (2 if m <= 16 else 1)   # (projection +) one fused launch
    y.backward(gy)
    got = [y.detach(), x.grad, A.grad, B.grad]
    x2, A2, B2 = (t.detach().clone().requires_grad_(True) for t in (x, A, B))

    def two_step():
        xl = x2 * mask if dropout else x2
        y2 = base(x2) + torch.nn.functional.linear(torch.nn.functional.linear(xl, A2), B2) * 0.25
        y2.backward(gy)
        return y2.detach()

    ref = [_unfused(q, two_step), x2.grad, A2.grad, B2.grad]
    for name, a_, b_ in zip(("y", "dx", "dA", "dB"), got, ref):
        assert a_.dtype == BF
        e = rel_err(np32(a_), np32(b_))
        assert e <= 4e-3, (name, e)


@pytest.mark.parametrize("dropout", [False, True])
def test_lora_group_matches_unfused(q, dropout):
    """`lora_linear4bit_group` (q/k/v: one launch per direction) over fp16 states vs three unfused two-step forms."""
    n_in, n_out, r = 512, 768, 32
    bases = [_linear(q, n_in, n_out, H16, bias=False, seed=i) for i in range(3)]
    As, Bs = _adapters(n_in, n_out, r, 3, seed=2)
    x = torch.randn(2, 150, n_in, device="cuda").to(BF).requires_grad_(True)
    gys = [torch.randn(2, 150, n_out, device="cuda").to(BF) for _ in range(3)]
    masks = [((torch.rand(2, 150, n_in, device="cuda") >= 0.1).float() / 0.9).to(BF) for _ in range(3)]
    assert q.lora._group_fusable(x, bases, As, Bs, None)
    xls = [x * mk for mk in masks] if dropout else None
    ys = q.lora_linear4bit_group(x, bases, As, Bs, 0.5, xls)
    torch.autograd.backward(ys, gys)
    got = [t.detach() for t in ys] + [x.grad] + [t.grad for t in As + Bs]
    x2 = x.detach().clone().requires_grad_(True)
    As2 = [t.detach().clone().requires_grad_(True) for t in As]
    Bs2 = [t.detach().clone().requires_grad_(True) for t in Bs]

    def two_step():
        ys2 = []
        for i in range(3):
            xl = x2 * masks[i] if dropout else x2
            ys2.append(bases[i](x2) + torch.nn.functional.linear(torch.nn.functional.linear(xl, As2[i]), Bs2[i]) * 0.5)
        torch.autograd.backward(ys2, gys)
        return [t.detach() for t in ys2]

    ref = _unfused(q, two_step) + [x2.grad] + [t.grad for t in As2 + Bs2]
    for idx, (a_, b_) in enumerate(zip(got, ref)):
        e = rel_err(np32(a_), np32(b_))
        # x.grad (idx 3) with dropout: autograd sums bf16 terms, 4 here (one grouped dX) and 6 in the reference (three dX)
        assert e <= (8e-3 if idx == 3 and dropout else 4e-3), (idx, e)


def test_lora_over_fp32_state_keeps_the_two_step_form(q):
    """Under bf16 compute an fp32 state's LoRA stays the two-step form, whose base call runs fused through Linear4bit."""
    F = q.functional
    base = _linear(q, 512, 768, F32, bias=False)
    (A,), (B,) = _adapters(512, 768, 16, 1, seed=4)
    x = act(40, 512, 6)
    assert not q.lora._group_fusable(x, [base], [A], [B], None)
    n0 = F.LAUNCH_COUNTER[0]
    y = base(x)
    assert F.LAUNCH_COUNTER[0] - n0 == 1
    y2 = y + torch.nn.functional.linear(torch.nn.functional.linear(x, A), B) * 0.5
    assert torch.equal(q.lora_linear4bit(x, base, A, B, 0.5), y2)


def test_lora_group_of_mixed_roundings_runs_per_linear(q):
    """An fp16 state next to a bf16 state under bf16 compute: not one launch, each linear runs fused on its own."""
    bases = [_linear(q, 256, 384, sd, bias=False, seed=i) for i, sd in enumerate((H16, BF))]
    As, Bs = _adapters(256, 384, 16, 2, seed=3)
    x = act(32, 256, 5)
    assert not q.lora._group_fusable(x, bases, As, Bs, None)
    assert all(q.lora._group_fusable(x, [b], [a], [bb], None) for b, a, bb in zip(bases, As, Bs))
    ys = q.lora_linear4bit_group(x, bases, As, Bs, 0.5)
    for i in range(2):
        assert torch.equal(ys[i], q.lora_linear4bit(x, bases[i], As[i], Bs[i], 0.5))


@pytest.mark.parametrize("state_dtype", [H16, F32])
def test_dora_over_fp16_and_fp32_states_keeps_the_peft_form(q, state_dtype):
    base = _linear(q, 256, 384, state_dtype, bias=False)
    (A,), (B,) = _adapters(256, 384, 16, 1, seed=6)
    mag = (torch.rand(384, device="cuda") + 0.5).to(BF)
    x = act(8, 256, 1)
    assert q.lora._group_fusable(x, [base], [A], [B], None) == (state_dtype == H16)
    assert not q.lora._dora_fusable(x, [base], [A], [B], [mag], None)
    assert torch.equal(q.lora.dora_linear4bit(x, base, A, B, mag, 0.5), q.lora.dora_linear4bit_peft(x, base, A, B, mag, 0.5))


# ---------------------------------------------------------------- HF path -------------------------------------------------

def test_hf_bf16_compute_over_fp16_checkpoint_in_fresh_interpreter():
    """BitsAndBytesConfig(nf4, double quant, bnb_4bit_compute_dtype=bf16) over an fp16 Llama model -> replace_with_bnb_linear:
    the state is fp16, the compute dtype bf16; a Linear4bit forward / backward in fp16 makes two fused launches and matches
    the oracle; the whole model's loss and backward run."""
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "shims") + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hf_mixed_case.py")], capture_output=True, text=True, env=env,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["bnb_file"].startswith(os.path.join(ROOT, "shims")) and out["n_linear4bit"] == 14
    assert out["compute_dtype"] == "torch.bfloat16" and out["state_dtype"] == "torch.float16"
    assert out["gpu_ok"] is True and out["fused_launches"] == 2 and out["backward_ok"] is True
