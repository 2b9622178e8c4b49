"""GPU parity of the fp16-compute fused path (`bnb_4bit_compute_dtype=torch.float16`, `qlora.py --fp16`).

The fused kernels dequantize to fp16_rn(LUT[j] * absmax): `dequantize_4bit(...).to(fp16)` for an fp16 or fp32 quant state.
Parity bar (DESIGN.md §2 with fp16 rounding): ||Y - Y_ref||_F / ||Y_ref||_F <= 1e-3 with both sides fp16-rounded, and every
element within one fp16 ulp (2^-10 of the binade of the largest magnitude) of the reference."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fp16_helpers import assert_close_f16, f16_round, np32, oracle_w16
from gpu_helpers import make_act, make_weight, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-3
H16 = torch.float16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def q():
    import qlora_b200 as q

    assert torch.cuda.is_available() and q._lib.load().qb200_has_fused_gemm() == 1
    return q


def act16(m, k, seed, scale=1.0):
    return (make_act(m, k, seed).float() * scale).to(H16)


def weight16(n, k, seed, scale=0.02):
    return make_weight(n, k, seed, dtype=H16, scale=scale)


def quantized(q, n, k, seed, nested=True, state_dtype=H16):
    w = make_weight(n, k, seed, dtype=state_dtype)
    packed, qs = q.functional.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
    assert qs.dtype == state_dtype
    return packed, qs


# ---------------------------------------------------------------- exact weights -------------------------------------------

@pytest.mark.parametrize("state_dtype", [H16, torch.float32])
@pytest.mark.parametrize("nested", [True, False])
def test_identity_reads_fp16_rounded_oracle_weights(q, c_oracle, nested, state_dtype):
    """Identity rows make each output one exact product 1.0 * w: forward must give W^T and dX must give W, equal bit for bit
    to the oracle's fp32 weight rounded to fp16 by numpy — and to `dequantize_4bit(...).to(fp16)`."""
    F = q.functional
    n, k = 384, 320
    packed, qs = quantized(q, n, k, seed=11, nested=nested, state_dtype=state_dtype)
    w16 = oracle_w16(c_oracle, packed, qs).astype(np.float16)
    y = F.nf4_linear_fwd(torch.eye(k, dtype=H16, device="cuda"), packed, qs)
    assert y.dtype == H16 and np.array_equal(y.cpu().numpy().view(np.uint16), np.ascontiguousarray(w16.T).view(np.uint16))
    dx = F.nf4_linear_bwd_dx(torch.eye(n, dtype=H16, device="cuda"), packed, qs)
    assert np.array_equal(dx.cpu().numpy().view(np.uint16), w16.view(np.uint16))
    wd = F.dequantize_4bit(packed, qs).to(H16)
    assert np.array_equal(wd.cpu().numpy().view(np.uint16), w16.view(np.uint16))
    # the skinny kernels read the same weights: one identity row at a time
    for i in (0, 63, k - 1):
        e = torch.zeros(1, k, dtype=H16, device="cuda")
        e[0, i] = 1
        assert np.array_equal(F.nf4_linear_fwd(e, packed, qs).cpu().numpy()[0].view(np.uint16), w16[:, i].view(np.uint16))


# ---------------------------------------------------------------- parity --------------------------------------------------

@pytest.mark.parametrize("state_dtype", [H16, torch.float32])
@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m,n,k", [(256, 128, 64), (300, 200, 192), (40, 96, 256), (512, 384, 1024)])
def test_fwd_bwd_small_shapes_vs_oracle(q, c_oracle, m, n, k, nested, state_dtype):
    F = q.functional
    packed, qs = quantized(q, n, k, seed=n * 7 + k, nested=nested, state_dtype=state_dtype)
    w = oracle_w16(c_oracle, packed, qs)
    x, dy = act16(m, k, 1), act16(m, n, 2)
    bias = weight16(1, n, seed=3, scale=0.5).view(-1)
    y = F.nf4_linear_fwd(x, packed, qs, bias)
    assert y.dtype == H16
    assert_close_f16(np32(y), f16_round(np32(x) @ w.T + np32(bias)))
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    assert_close_f16(np32(dx), f16_round(np32(dy) @ w))
    # fp32 output: the fp16-rounded result, widened
    assert torch.equal(F.nf4_linear_fwd(x, packed, qs, bias, out_dtype=torch.float32), y.float())
    assert torch.equal(F.nf4_linear_bwd_dx(dy, packed, qs, out_dtype=torch.float32), dx.float())


# Llama-2-7B, Llama-2-13B and LLaMA-65B linear shapes
MODEL_SHAPES = [(4096, 4096), (11008, 4096), (4096, 11008), (5120, 5120), (13824, 5120), (5120, 13824),
                (8192, 8192), (22016, 8192), (8192, 22016)]


@pytest.mark.parametrize("n,k", MODEL_SHAPES)
def test_model_shapes_vs_fp32_reference(q, n, k):
    """Forward and dX at the model shapes against an fp32 GEMM over the exact fp16 weights (the identity test shows they
    are the oracle's), rounded to fp16 once."""
    F = q.functional
    m = 512
    packed, qs = quantized(q, n, k, seed=n ^ k)
    wd = F.dequantize_4bit(packed, qs).float()
    x, dy = act16(m, k, 3), act16(m, n, 4)
    y = F.nf4_linear_fwd(x, packed, qs)
    assert_close_f16(np32(y), np32((x.float() @ wd.t()).half()))
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    assert_close_f16(np32(dx), np32((dy.float() @ wd).half()))
    assert torch.equal(F.nf4_linear_fwd(x, packed, qs), y) and torch.equal(F.nf4_linear_bwd_dx(dy, packed, qs), dx)


@pytest.mark.parametrize("m", [17, 48, 80, 300, 768])
def test_split_k_vs_oracle(q, c_oracle, m):
    """17..768 tokens: the split-K schedule (fp32 partials in a lent workspace + the fp16 reduce) where the library plans it,
    forward with bias and dX, plain and with LoRA operands."""
    F = q.functional
    lib = q._lib.load()
    n, k, r = 2048, 4096, 64
    if m <= 48:
        assert lib.qb200_nf4_linear_workspace_size(m, n, k, 1) > 0
    packed, qs = quantized(q, n, k, seed=77)
    w = oracle_w16(c_oracle, packed, qs)
    x, dy = act16(m, k, 1), act16(m, n, 2)
    bias = weight16(1, n, seed=3, scale=0.5).view(-1)
    assert_close_f16(np32(F.nf4_linear_fwd(x, packed, qs, bias)), f16_round(np32(x) @ w.T + np32(bias)))
    assert_close_f16(np32(F.nf4_linear_bwd_dx(dy, packed, qs)), f16_round(np32(dy) @ w))
    u, v, a = act16(m, r, 4, 0.5), weight16(n, r, 5, 0.2), weight16(r, k, 6, 0.2)
    assert_close_f16(np32(F.nf4_linear_fwd_lora(x, packed, qs, u, v)), f16_round(np32(x) @ w.T + np32(u) @ np32(v).T))
    assert_close_f16(np32(F.nf4_linear_bwd_dx_lora(dy, packed, qs, u, a)), f16_round(np32(dy) @ w + np32(u) @ np32(a)))
    # fp32 output through the reduce: the fp16-rounded sum, widened
    assert torch.equal(F.nf4_linear_fwd(x, packed, qs, bias, out_dtype=torch.float32), F.nf4_linear_fwd(x, packed, qs, bias).float())


@pytest.mark.parametrize("m,n,k", [(2048, 512, 256), (1500, 768, 512)])
def test_range_schedule_units_bit_equal_across_token_counts(q, m, n, k):
    F = q.functional
    lib = q._lib.load()
    packed, qs = quantized(q, n, k, seed=9)
    x, dy = act16(m, k, 5), act16(m, n, 6)
    y, dx = F.nf4_linear_fwd(x, packed, qs), F.nf4_linear_bwd_dx(dy, packed, qs)
    for m2 in (m // 2 + 8, m - 16, 800, 112, 333):
        for is_bwd, full, inp in ((0, y, x), (1, dx, dy)):
            part = (F.nf4_linear_bwd_dx if is_bwd else F.nf4_linear_fwd)(inp[:m2].contiguous(), packed, qs)
            if lib.qb200_nf4_linear_workspace_size(m2, n, k, is_bwd) == 0:
                assert torch.equal(part, full[:m2]), (m2, is_bwd)
            else:
                assert_close_f16(np32(part), np32(full[:m2]))


@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m,n,k,r,nprob", [(300, 200, 192, 16, 3), (2047, 512, 1024, 64, 2), (17, 128, 128, 0, 3), (9, 384, 320, 16, 3),
                                           (1, 256, 128, 64, 2), (700, 1032, 320, 32, 3)])
def test_grouped_launches_vs_oracle_and_per_linear(q, c_oracle, m, n, k, r, nprob, nested):
    """q/k/v (3) and gate/up (2) as one launch per direction: forward outputs as column slices of one buffer (strided U
    too), the backward contraction sum; the grouped dX equals the sum of per-linear launches within the bar."""
    F = q.functional
    packs, states, ws = [], [], []
    for i in range(nprob):
        packed, qs = quantized(q, n, k, seed=31 * i + n + k, nested=nested, state_dtype=(H16, torch.float32)[i % 2])
        packs.append(packed.t())
        states.append(qs)
        ws.append(oracle_w16(c_oracle, packed, qs))
    x = act16(m, k, 1)
    us = vs = gs = as_ = None
    if r:
        u_cat = act16(m, nprob * r, 2, 0.5)
        us = [u_cat[:, i * r:(i + 1) * r] for i in range(nprob)]
        vs = [weight16(n, r, 20 + i, 0.2) for i in range(nprob)]
        gs = [act16(m, r, 40 + i, 0.5) for i in range(nprob)]
        as_ = [weight16(r, k, 50 + i, 0.2) for i in range(nprob)]
    out_cat = torch.full((m, nprob * n), float("nan"), device="cuda", dtype=H16)
    outs = [out_cat[:, i * n:(i + 1) * n] for i in range(nprob)]
    ys = F.nf4_linear_group(False, [x] * nprob, packs, states, us=us, vs=vs, outs=outs)
    for i in range(nprob):
        ref = np32(x) @ ws[i].T + (np32(us[i]) @ np32(vs[i]).T if r else 0.0)
        assert ys[i].data_ptr() == outs[i].data_ptr()
        assert_close_f16(np32(ys[i]), f16_round(ref))
    assert not torch.isnan(out_cat.float()).any()
    dys = [act16(m, n, 30 + i) for i in range(nprob)]
    dx = F.nf4_linear_group(True, dys, packs, states, us=gs, vs=as_)
    acc = sum(np32(dys[i]) @ ws[i] + (np32(gs[i]) @ np32(as_[i]) if r else 0.0) for i in range(nprob))
    assert_close_f16(np32(dx), f16_round(acc))
    # the per-linear sum carries one fp16 rounding per linear: one ulp each
    per = sum(F.nf4_linear_group(True, [dys[i]], [packs[i]], [states[i]], us=None if not r else [gs[i]],
                                 vs=None if not r else [as_[i]], out_dtype=torch.float32) for i in range(nprob))
    assert_close_f16(np32(dx), np32(per), ulps=nprob)


# ---------------------------------------------------------------- skinny kernels ------------------------------------------

@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m", [1, 2, 5, 8, 9, 16, 17, 24, 32])
@pytest.mark.parametrize("n,k", [(4096, 4096), (200, 192), (24, 320), (4096, 11008)])
def test_skinny_forward_up_to_32_tokens(q, c_oracle, m, n, k, nested):
    """1..16 tokens run the fp16 skinny kernels, 17..32 cross into the wgmma kernel: bias, pitched input and output."""
    F = q.functional
    packed, qs = quantized(q, n, k, seed=3 * n + k, nested=nested)
    w = oracle_w16(c_oracle, packed, qs)
    x_wide = act16(m, k + 64, 10 + m)
    x = x_wide[:, :k]                                       # row pitch k + 64
    bias = weight16(1, n, 9, 0.5).view(-1)
    for b in (bias, None):
        out_cat = torch.full((m, n + 8), float("nan"), device="cuda", dtype=H16)
        y = F.nf4_linear_group(False, [x], [packed], [qs], None if b is None else [b], outs=[out_cat[:, :n]])[0]
        ref = np32(x) @ w.T + (np32(b) if b is not None else 0.0)
        assert_close_f16(np32(y), f16_round(ref))
        assert torch.isnan(out_cat[:, n:].float()).all()


@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m,r", [(1, 64), (1, 8), (3, 16), (8, 64), (16, 24)])
@pytest.mark.parametrize("n,k", [(4096, 4096), (200, 192)])
def test_skinny_forward_with_lora_operands(q, c_oracle, m, r, n, k, nested):
    F = q.functional
    packed, qs = quantized(q, n, k, seed=7 * n + k, nested=nested, state_dtype=torch.float32)
    w = oracle_w16(c_oracle, packed, qs)
    x = act16(m, k, 20 + m)
    u = act16(m, r + 8, 21 + r)[:, :r]                      # row pitch r + 8
    v = weight16(n, r, 22 + r, 0.05)
    bias = weight16(1, n, 9, 0.5).view(-1)
    assert q._lib.load().qb200_nf4_linear_workspace_size(m, n, k, 0) == 0
    for b in (None, bias):
        y = F.nf4_linear_fwd_lora(x, packed, qs, u, v, b)
        ref = np32(x) @ w.T + np32(u) @ np32(v).T + (np32(b) if b is not None else 0.0)
        assert_close_f16(np32(y), f16_round(ref))


@pytest.mark.parametrize("m", [1, 4, 16])
def test_skinny_grouped_forward_pdl_chain(q, m):
    """A decode chain of grouped fp16 forwards (one skinny launch per problem, chained by programmatic dependent launch),
    each reading the previous launch's output and weights quantized one launch earlier, equals the same launches with a
    synchronize between them."""
    F = q.functional
    n = k = 2048
    x0 = act16(m, k, 70, 0.5)
    for it in range(3):
        pq = [quantized(q, n, k, seed=100 + 3 * it + i) for i in range(3)]
        packs, states = [p.t() for p, _ in pq], [s for _, s in pq]

        def step(x):
            return F.nf4_linear_group(False, [x] * 3, packs, states)

        ys1 = step(x0)
        ys2 = step(ys1[2])
        torch.cuda.synchronize()
        r1 = step(x0)
        torch.cuda.synchronize()
        r2 = step(r1[2])
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(ys1 + ys2, r1 + r2))


@pytest.mark.parametrize("m", [1, 3, 8, 16])
@pytest.mark.parametrize("k,r", [(4096, 64), (11008, 192), (320, 8)])
def test_typed_lora_project(q, m, k, r):
    """`qb200_lora_project_typed` in fp16: U = s * x . A^T against fp32 numpy and `torch.addmm(..., alpha=s)` in fp16."""
    F = q.functional
    a = weight16(r, k, r + k, 0.05)
    x_wide = act16(m, k + 64, m + k)
    ref = f16_round((np32(x_wide[:, :k]) @ np32(a).T) * np.float32(0.25))
    for x in (x_wide[:, :k].contiguous(), x_wide[:, :k]):
        u = F.lora_project(x, a, 0.25)
        assert u.shape == (m, r) and u.dtype == H16
        assert_close_f16(np32(u), ref)
    u_mm = torch.addmm(torch.empty(m, r, dtype=H16, device="cuda"), x_wide[:, :k].contiguous(), a.t(), beta=0.0, alpha=0.25)
    assert_close_f16(np32(F.lora_project(x_wide[:, :k], a, 0.25)), np32(u_mm))


# ---------------------------------------------------------------- module, autograd, fp32 fold ------------------------------

def _linear16(q, n_in, n_out, state_dtype, bias=False, seed=0):
    torch.manual_seed(seed)
    lin = q.nn.Linear4bit(n_in, n_out, bias=bias, compute_dtype=H16, compress_statistics=True, quant_type="nf4")
    lin.weight.data = lin.weight.data.to(state_dtype)
    if bias:
        lin.bias.data = (torch.randn(n_out) * 0.1)
    lin = lin.cuda()
    assert lin.weight.quant_state.dtype == state_dtype
    return lin


@pytest.mark.parametrize("state_dtype", [H16, torch.float32])
def test_module_fp16_compute_vs_oracle(q, c_oracle, state_dtype):
    """Linear4bit(compute_dtype=fp16) over an fp16 / fp32 state, fp16 activations: fused forward and backward."""
    F = q.functional
    lin = _linear16(q, 256, 384, state_dtype, bias=True)
    w = oracle_w16(c_oracle, lin.weight.data, lin.weight.quant_state)
    x = act16(100, 256, 1).view(2, 50, 256).requires_grad_(True)
    n0 = F.LAUNCH_COUNTER[0]
    y = lin(x)
    assert y.dtype == H16 and y.shape == (2, 50, 384)
    gy = act16(100, 384, 2).view(2, 50, 384)
    y.backward(gy)
    assert F.LAUNCH_COUNTER[0] - n0 == 2                    # one fused launch per direction, no dequantize
    b = np32(lin.bias.to(H16))
    assert_close_f16(np32(y).reshape(100, 384), f16_round(np32(x).reshape(100, 256) @ w.T + b))
    assert_close_f16(np32(x.grad).reshape(100, 256), f16_round(np32(gy).reshape(100, 384) @ w))
    assert rel_err(np32(lin.bias.grad), np32(gy).reshape(100, 384).sum(0)) <= 2e-3


@pytest.mark.parametrize("state_dtype", [H16, torch.float32])
def test_fp32_activations_fold_into_the_fp16_fused_node(q, state_dtype):
    """`qlora.py --fp16`: fp32 activations, fp16 compute, fp32 out.  Forward gives exactly the fp16 fused output widened,
    the input gradient exactly the fp16 fused dX widened."""
    F = q.functional
    lin = _linear16(q, 512, 768, state_dtype, bias=True)
    qs, packed = lin.weight.quant_state, lin.weight.data
    x = torch.randn(3, 40, 512, device="cuda", requires_grad=True)
    y = lin(x)
    assert y.dtype == torch.float32
    y16 = F.nf4_linear_fwd(x.detach().half().view(-1, 512), packed, qs, lin.bias.detach().half())
    assert torch.equal(y.detach().view(-1, 768), y16.float())
    gy = torch.randn_like(y)
    y.backward(gy)
    assert x.grad.dtype == torch.float32
    assert torch.equal(x.grad.view(-1, 512), F.nf4_linear_bwd_dx(gy.half().view(-1, 768), packed, qs).float())


def test_bf16_state_with_fp16_compute_stays_unfused(q):
    """A bf16 state under fp16 compute would round twice: it keeps today's dequantize + cuBLAS path, bit for bit."""
    lin = _linear16(q, 256, 384, torch.bfloat16)
    x = act16(64, 256, 1).requires_grad_(True)
    gy = act16(64, 384, 2)
    y = lin(x)
    y.backward(gy)
    got = (y.detach().clone(), x.grad.clone())
    x.grad = None
    q.autograd.USE_FUSED = False
    try:
        y2 = lin(x)
        y2.backward(gy)
    finally:
        q.autograd.USE_FUSED = True
    assert torch.equal(got[0], y2) and torch.equal(got[1], x.grad)


# ---------------------------------------------------------------- LoRA -----------------------------------------------------

def _adapters(n_in, n_out, r, count, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    As = [(torch.randn(r, n_in, generator=g) * 0.05).to(H16).cuda().requires_grad_(True) for _ in range(count)]
    Bs = [(torch.randn(n_out, r, generator=g) * 0.05).to(H16).cuda().requires_grad_(True) for _ in range(count)]
    return As, Bs


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("m", [4, 300])
def test_lora_linear4bit_fp16_matches_unfused(q, dropout, m):
    """`lora_linear4bit` with an fp16 base (fp32 state), fp16 adapters and fp16 x, fused, against peft's two-step form."""
    F = q.functional
    base = _linear16(q, 512, 768, torch.float32)
    (A,), (B,) = _adapters(512, 768, 64, 1, seed=1)
    x = act16(m, 512, 3).view(1, m, 512).requires_grad_(True)
    gy = act16(m, 768, 4).view(1, m, 768)
    mask = ((torch.rand(1, m, 512, device="cuda") >= 0.1).float() / 0.9).to(H16)
    assert q.lora._group_fusable(x, [base], [A], [B], None)
    n0 = F.LAUNCH_COUNTER[0]
    y = q.lora_linear4bit(x, base, A, B, 0.25, x_lora=x * mask if dropout else None)
    assert F.LAUNCH_COUNTER[0] - n0 == (2 if m <= 16 else 1)   # (projection +) one fused launch
    y.backward(gy)
    got = [y.detach(), x.grad, A.grad, B.grad]
    x2, A2, B2 = (t.detach().clone().requires_grad_(True) for t in (x, A, B))
    xl = x2 * mask if dropout else x2
    y2 = base(x2) + torch.nn.functional.linear(torch.nn.functional.linear(xl, A2), B2) * 0.25
    y2.backward(gy)
    for name, a_, b_ in zip(("y", "dx", "dA", "dB"), got, [y2.detach(), x2.grad, A2.grad, B2.grad]):
        assert a_.dtype == H16
        e = rel_err(np32(a_), np32(b_))
        assert e <= 4e-3, (name, e)


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("x_dtype", [H16, torch.float32])
def test_lora_group_fp16_matches_per_linear_and_unfused(q, dropout, x_dtype):
    """`lora_linear4bit_group` (q/k/v: one launch per direction) in fp16 vs three unfused two-step forms."""
    n_in, n_out, r = 512, 768, 32
    bases = [_linear16(q, n_in, n_out, (H16, torch.float32)[i % 2], seed=i) for i in range(3)]
    As, Bs = _adapters(n_in, n_out, r, 3, seed=2)
    x = torch.randn(2, 150, n_in, device="cuda").to(x_dtype).requires_grad_(True)
    gys = [torch.randn(2, 150, n_out, device="cuda").to(x_dtype) for _ in range(3)]
    masks = [((torch.rand(2, 150, n_in, device="cuda") >= 0.1).float() / 0.9).to(H16) for _ in range(3)]
    assert q.lora._group_fusable(x, bases, As, Bs, None)
    xls = [x.to(H16) * mk for mk in masks] if dropout else None
    ys = q.lora_linear4bit_group(x, bases, As, Bs, 0.5, xls)
    torch.autograd.backward(ys, gys)
    got = [t.detach() for t in ys] + [x.grad] + [t.grad for t in As + Bs]
    assert all(y.dtype == x_dtype for y in ys) and x.grad.dtype == x_dtype
    x2 = x.detach().clone().requires_grad_(True)
    As2 = [t.detach().clone().requires_grad_(True) for t in As]
    Bs2 = [t.detach().clone().requires_grad_(True) for t in Bs]
    ys2 = []
    for i in range(3):
        xl = x2.to(H16) * masks[i] if dropout else x2.to(H16)
        upd = torch.nn.functional.linear(torch.nn.functional.linear(xl, As2[i]), Bs2[i]) * 0.5
        ys2.append(bases[i](x2) + upd.to(x_dtype))
    torch.autograd.backward(ys2, gys)
    ref = [t.detach() for t in ys2] + [x2.grad] + [t.grad for t in As2 + Bs2]
    for idx, (a_, b_) in enumerate(zip(got, ref)):
        e = rel_err(np32(a_), np32(b_))
        assert e <= 4e-3, (idx, e)


def test_fp16_lora_cuda_graph_replay_equals_eager(q):
    base = _linear16(q, 512, 1024, H16)
    (A,), (B,) = _adapters(512, 1024, 16, 1, seed=5)
    x_static = torch.randn(700, 512, device="cuda", dtype=H16).requires_grad_(True)
    gy = torch.randn(700, 1024, device="cuda", dtype=H16)

    def fwd_bwd():
        for t in (x_static, A, B):
            t.grad = None
        y = q.lora_linear4bit(x_static, base, A, B, 0.5)
        y.backward(gy)
        return y.detach(), x_static.grad, A.grad, B.grad

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


def test_dora_with_fp16_keeps_the_peft_form(q):
    base = _linear16(q, 256, 384, torch.float32)
    (A,), (B,) = _adapters(256, 384, 16, 1, seed=6)
    mag = torch.ones(384, device="cuda", dtype=H16)
    x = act16(8, 256, 1)
    assert not q.lora._dora_fusable(x, [base], [A], [B], [mag], None)
    assert torch.equal(q.lora.dora_linear4bit(x, base, A, B, mag, 0.5), q.lora.dora_linear4bit_peft(x, base, A, B, mag, 0.5))


# ---------------------------------------------------------------- HF path -------------------------------------------------

def test_hf_fp16_compute_path_in_fresh_interpreter():
    """BitsAndBytesConfig(nf4, double quant, bnb_4bit_compute_dtype=fp16) -> replace_with_bnb_linear -> an fp16 model:
    a Linear4bit forward / backward against the oracle and the whole model's loss, in a fresh interpreter."""
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "shims") + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hf_fp16_case.py")], capture_output=True, text=True, env=env,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["bnb_file"].startswith(os.path.join(ROOT, "shims")) and out["n_linear4bit"] == 14
    assert out["compute_dtype"] == "torch.float16" and out["state_dtype"] == "torch.float16"
    assert out["gpu_ok"] is True and out["fused_launches"] == 2
