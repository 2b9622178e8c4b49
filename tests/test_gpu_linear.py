"""GPU parity: fused NF4 dequant + wgmma GEMM (forward and dX) vs the oracle.

Tolerance (north_star: "within 1e-3 relative bf16"): ||Y - Y_ref||_F / ||Y_ref||_F <= 1e-3 with both sides
bf16-rounded, AND every element within one bf16 ulp (2^-8 of the largest magnitude) of the reference —
summation order differs between wgmma, cuBLAS and the CPU, so an fp32 accumulator can round to the
adjacent bf16 value (a max-norm bound below one ulp is unattainable for ANY bf16 GEMM, cuBLAS included).
The dequantized weights feeding the tensor core ARE bit-exact (identity-input test below)."""
import numpy as np
import pytest
import torch

import oracle_c as oc
from gpu_helpers import assert_close_bf16, bf16_to_f32_np, make_act, make_weight, rel_err, state_to_numpy
from oracle import nf4_oracle as o

pytestmark = pytest.mark.gpu
TOL = 1e-3


@pytest.fixture(scope="module")
def q():
    import qlora_b200 as q

    assert torch.cuda.is_available()
    from qlora_b200 import _lib

    lib = _lib.load()
    assert lib.qb200_has_fused_gemm() == 1
    return q


def _oracle_weight(packed, qs, c_oracle):
    st = state_to_numpy(packed, qs)
    n = int(np.prod(st["shape"]))
    if st["nested"]:
        w = oc.dequantize_nested_to_f32(c_oracle, st["packed"], st["absmax_u8"], st["code256"], st["absmax2"], st["offset"], n)
    else:
        bits = oc.dequantize_nf4_bf16_bits(c_oracle, st["packed"], st["absmax"], n)
        w = (bits.astype(np.uint32) << 16).view(np.float32)
    return w.reshape(st["shape"])


@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m,n,k", [(256, 128, 64), (256, 128, 256), (40, 96, 256), (300, 200, 192), (1, 128, 128),
                                   (512, 384, 1024), (2048, 512, 4096)])
def test_fused_fwd_bwd_vs_oracle(q, c_oracle, m, n, k, nested):
    F = q.functional
    w = make_weight(n, k, seed=n * 7 + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    x = make_act(m, k, seed=1)
    y = F.nf4_linear_fwd(x, packed, qs)
    y_ref = o.bf16_round(bf16_to_f32_np(x) @ w_ref.T)
    assert y.shape == (m, n) and y.dtype == torch.bfloat16
    assert_close_bf16(bf16_to_f32_np(y), y_ref, TOL)
    dy = make_act(m, n, seed=2)
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    dx_ref = o.bf16_round(bf16_to_f32_np(dy) @ w_ref)
    assert dx.shape == (m, k)
    assert_close_bf16(bf16_to_f32_np(dx), dx_ref, TOL)


def test_fused_reads_bit_exact_weights(q, c_oracle):
    """Feeding identity rows makes each output ONE product 1.0 * w (exact in fp32, bf16 in -> bf16 out),
    so Y must equal the oracle's dequantized bf16 weight bit for bit — forward reads W^T, dX reads W."""
    F = q.functional
    n, k = 384, 320
    w = make_weight(n, k, seed=11)
    packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    eye_k = torch.eye(k, dtype=torch.bfloat16, device="cuda")
    y = F.nf4_linear_fwd(eye_k, packed, qs)          # [k, n] = W^T
    assert np.array_equal(bf16_to_f32_np(y).view(np.uint32), np.ascontiguousarray(w_ref.T).view(np.uint32))
    eye_n = torch.eye(n, dtype=torch.bfloat16, device="cuda")
    dx = F.nf4_linear_bwd_dx(eye_n, packed, qs)      # [n, k] = W
    assert np.array_equal(bf16_to_f32_np(dx).view(np.uint32), w_ref.view(np.uint32))


def test_golden_linear(q, golden):
    F = q.functional
    g = golden
    packed = torch.from_numpy(g["A_packed"]).cuda().view(-1, 1)
    st2 = F.QuantState(absmax=torch.from_numpy(g["A_absmax2"]).cuda(), code=torch.from_numpy(g["code256"]).cuda(), blocksize=256, dtype=torch.float32)
    qs = F.QuantState(absmax=torch.from_numpy(g["A_absmax_u8"]).cuda(), shape=torch.Size(g["A_w"].shape), dtype=torch.bfloat16, blocksize=64,
                      quant_type="nf4", code=F.get_4bit_type("nf4"), offset=torch.tensor(float(g["A_offset"]), device="cuda"), state2=st2)
    x = torch.from_numpy(g["A_x"]).cuda().to(torch.bfloat16)
    dy = torch.from_numpy(g["A_dy"]).cuda().to(torch.bfloat16)
    assert_close_bf16(bf16_to_f32_np(F.nf4_linear_fwd(x, packed, qs)), g["A_y"], TOL)
    assert_close_bf16(bf16_to_f32_np(F.nf4_linear_bwd_dx(dy, packed, qs)), g["A_dx"], TOL)


@pytest.mark.parametrize("n,k", [(4096, 4096), (11008, 4096), (4096, 11008)])
def test_full_size_vs_unfused_and_properties(q, n, k):
    """BASELINE.json full sizes (M = 2048): compare with the unfused GPU path (our bit-exact dequant
    kernel + cuBLAS) and check linearity, which does not need a CPU GEMM."""
    F = q.functional
    m = 2048
    w = make_weight(n, k, seed=n + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
    wd = F.dequantize_4bit(packed, qs)  # bit-exact vs oracle (test_gpu_quant)
    x = make_act(m, k, seed=3)
    y = F.nf4_linear_fwd(x, packed, qs)
    y_ref = (x.float() @ wd.float().t()).to(torch.bfloat16).float()
    assert_close_bf16(y.float().cpu().numpy(), y_ref.cpu().numpy(), TOL)
    dy = make_act(m, n, seed=4)
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    dx_ref = (dy.float() @ wd.float()).to(torch.bfloat16).float()
    assert_close_bf16(dx.float().cpu().numpy(), dx_ref.cpu().numpy(), TOL)
    # linearity in the activation: f(2x) == 2 f(x) exactly (power-of-two scaling commutes with rounding)
    y2 = F.nf4_linear_fwd((x * 2).contiguous(), packed, qs)
    assert torch.equal(y2, y * 2)
    # determinism
    assert torch.equal(F.nf4_linear_fwd(x, packed, qs), y)


def test_module_autograd_and_dtypes(q, c_oracle):
    """Linear4bit forward/backward through autograd: fp32 input (as from qlora.py:400-401's fp32 norms)
    is computed in bf16 and returned as fp32; grads flow to x and bias only (SURVEY.md 8a a7/a11)."""
    torch.manual_seed(0)
    lin = q.nn.Linear4bit(256, 384, bias=True, compute_dtype=torch.bfloat16, compress_statistics=True, quant_type="nf4")
    w0 = lin.weight.data.clone()
    lin = lin.cuda()
    assert lin.weight.dtype == torch.uint8 and lin.weight.shape == (256 * 384 // 2, 1) and lin.weight.quant_state.nested
    w_ref = _oracle_weight(lin.weight.data, lin.weight.quant_state, c_oracle)
    # weight was quantized from the fp32 init: round trip close to the original
    assert np.abs(w_ref - w0.numpy()).mean() < 0.1 * np.abs(w0.numpy()).mean() + 1e-3
    x = torch.randn(2, 50, 256, device="cuda", requires_grad=True)
    y = lin(x)
    assert y.dtype == torch.float32 and y.shape == (2, 50, 384)
    xb = o.bf16_round(x.detach().cpu().numpy().reshape(-1, 256))
    bias = o.bf16_round(lin.bias.detach().float().cpu().numpy())
    y_ref = o.bf16_round(xb @ w_ref.T + bias)
    assert_close_bf16(y.detach().cpu().numpy().reshape(-1, 384), y_ref, TOL)
    gy = torch.randn_like(y)
    y.backward(gy)
    gyb = o.bf16_round(gy.cpu().numpy().reshape(-1, 384))
    assert_close_bf16(x.grad.cpu().numpy().reshape(-1, 256), o.bf16_round(gyb @ w_ref), TOL)
    assert lin.weight.grad is None
    assert rel_err(lin.bias.grad.float().cpu().numpy(), gyb.sum(0)) <= 2e-2
    # the unfused GPU path (fp16 compute dtype is not covered by the fused kernel) agrees too
    lin16 = q.nn.Linear4bit(256, 384, bias=False, compute_dtype=torch.float16, quant_type="nf4")
    lin16.weight = lin.weight
    y16 = lin16(x.detach().half())
    assert y16.dtype == torch.float16
    w16 = w_ref.astype(np.float16).astype(np.float32)
    assert rel_err(y16.float().cpu().numpy().reshape(-1, 384), x.detach().half().float().cpu().numpy().reshape(-1, 256) @ w16.T) <= 2e-3


def test_state_dict_roundtrip(q):
    lin = q.nn.Linear4bit(128, 64, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4").cuda()
    sd = lin.state_dict()
    assert set(sd) == {"weight", "weight.absmax", "weight.quant_map", "weight.nested_absmax", "weight.nested_quant_map",
                       "weight.quant_state.bitsandbytes__nf4"}
    lin2 = q.nn.Linear4bit(128, 64, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
    lin2.load_state_dict(sd)
    x = torch.randn(8, 128, device="cuda", dtype=torch.bfloat16)
    assert torch.equal(lin(x), lin2(x))
    # from_prequantized, the HF loading path
    stats = {k[len("weight."):]: v for k, v in sd.items() if k != "weight"}
    p = q.nn.Params4bit.from_prequantized(sd["weight"], stats, device="cuda")
    assert p.quant_state.nested and p.quant_state.shape == torch.Size([64, 128])


@pytest.mark.parametrize("m,n,k,r", [(256, 256, 256, 64), (300, 200, 192, 16), (2048, 512, 1024, 64), (1000, 640, 512, 8)])
def test_fused_lora_step_vs_oracle(q, c_oracle, m, n, k, r):
    """SURVEY.md 8f-1: Y = X.W^T + U.V^T and dX = dY.W + U.Vt in ONE launch (extra bf16 contraction step)."""
    F = q.functional
    w = make_weight(n, k, seed=n + k + r)
    packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    x, dy = make_act(m, k, seed=1), make_act(m, n, seed=2)
    u = (make_act(m, r, seed=3).float() * 0.5).to(torch.bfloat16)
    v = make_weight(n, r, seed=4, scale=0.2)          # lora_B.weight  [N, r]
    g = (make_act(m, r, seed=5).float() * 0.5).to(torch.bfloat16)
    a = make_weight(r, k, seed=6, scale=0.2)          # lora_A.weight  [r, K]
    y = F.nf4_linear_fwd_lora(x, packed.t(), qs, u, v)
    y_ref = o.bf16_round(bf16_to_f32_np(x) @ w_ref.T + bf16_to_f32_np(u) @ bf16_to_f32_np(v).T)
    assert_close_bf16(bf16_to_f32_np(y), y_ref, TOL)
    dx = F.nf4_linear_bwd_dx_lora(dy, packed.t(), qs, g, a)
    dx_ref = o.bf16_round(bf16_to_f32_np(dy) @ w_ref + bf16_to_f32_np(g) @ bf16_to_f32_np(a))
    assert_close_bf16(bf16_to_f32_np(dx), dx_ref, TOL)
    # the update alone: zero activations isolate U.V^T (exact products of bf16 pairs, fp32 accumulate)
    y0 = F.nf4_linear_fwd_lora(torch.zeros_like(x), packed.t(), qs, u, v)
    assert_close_bf16(bf16_to_f32_np(y0), o.bf16_round(bf16_to_f32_np(u) @ bf16_to_f32_np(v).T), TOL)


def test_fused_lora_autograd_matches_unfused(q):
    """`lora_linear4bit` (fused: LoraMatMul4Bit with one linear) vs peft's two-step form built from the same kernels: outputs
    and all gradients."""
    torch.manual_seed(0)
    base = q.nn.Linear4bit(512, 768, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4").cuda()
    A = (torch.randn(64, 512, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    B = (torch.randn(768, 64, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    x = torch.randn(3, 100, 512, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    gy = torch.randn(3, 100, 768, device="cuda", dtype=torch.bfloat16)
    y = q.lora_linear4bit(x, base, A, B, 0.25)
    y.backward(gy)
    got = [y.detach().float(), x.grad.float(), A.grad.float(), B.grad.float()]
    x2, A2, B2 = (t.detach().clone().requires_grad_(True) for t in (x, A, B))
    y2 = base(x2) + torch.nn.functional.linear(torch.nn.functional.linear(x2, A2), B2) * 0.25
    y2.backward(gy)
    ref = [y2.detach().float(), x2.grad.float(), A2.grad.float(), B2.grad.float()]
    for name, a_, b_ in zip(("y", "dx", "dA", "dB"), got, ref):
        e = rel_err(a_.cpu().numpy(), b_.cpu().numpy())
        assert e <= 4e-3, (name, e)   # two bf16 roundings in the reference sequence vs one in the fused kernel
    assert y.shape == (3, 100, 768) and base.weight.grad is None


@pytest.mark.parametrize("m", [1, 16, 48, 64, 80, 300, 512, 1024])
def test_small_m_split_k(q, c_oracle, m):
    """Small token counts: the split-K schedule (fp32 partials in a lent workspace + reduce) for the smallest, the range
    schedule with few-token units (wgmma N = 16..) above — forward with bias, dX, and the fused-LoRA forms, all against
    the oracle.  The library decides (qb200_nf4_linear_workspace_size > 0 <=> split-K)."""
    F = q.functional
    from qlora_b200 import _lib

    n, k, r = 2048, 4096, 64
    ws = _lib.load().qb200_nf4_linear_workspace_size(m, n, k, 0)
    ws_b = _lib.load().qb200_nf4_linear_workspace_size(m, n, k, 1)
    assert ws >= 0 and ws_b >= 0 and (ws == 0 if m <= 4 else True)  # few-token forward is the skinny kernel
    if m <= 16:
        assert ws_b > 0   # the smallest token counts really are split
    w = make_weight(n, k, seed=77)
    packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    x, dy = make_act(m, k, seed=1), make_act(m, n, seed=2)
    bias = make_weight(1, n, seed=3, scale=0.5).view(-1)
    y = F.nf4_linear_fwd(x, packed, qs, bias)
    y_ref = o.bf16_round(bf16_to_f32_np(x) @ w_ref.T + bf16_to_f32_np(bias))
    assert_close_bf16(bf16_to_f32_np(y), y_ref, TOL)
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    assert_close_bf16(bf16_to_f32_np(dx), o.bf16_round(bf16_to_f32_np(dy) @ w_ref), TOL)
    u = (make_act(m, r, seed=4).float() * 0.5).to(torch.bfloat16)
    v = make_weight(n, r, seed=5, scale=0.2)
    a = make_weight(r, k, seed=6, scale=0.2)
    yl = F.nf4_linear_fwd_lora(x, packed.t(), qs, u, v)
    assert_close_bf16(bf16_to_f32_np(yl), o.bf16_round(bf16_to_f32_np(x) @ w_ref.T + bf16_to_f32_np(u) @ bf16_to_f32_np(v).T), TOL)
    dxl = F.nf4_linear_bwd_dx_lora(dy, packed.t(), qs, u, a)
    assert_close_bf16(bf16_to_f32_np(dxl), o.bf16_round(bf16_to_f32_np(dy) @ w_ref + bf16_to_f32_np(u) @ bf16_to_f32_np(a)), TOL)
    # empty batch
    assert F.nf4_linear_fwd(x[:0], packed, qs).shape == (0, n)


@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
@pytest.mark.parametrize("n,k", [(4096, 4096), (11008, 4096), (200, 192)])
def test_gemv_small_batch(q, c_oracle, m, n, k, nested):
    """SURVEY.md 8f-2: single-/few-token forward (the generation path) runs the weight-streaming skinny kernel."""
    F = q.functional
    w = make_weight(n, k, seed=5 * n + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    x = make_act(m, k, seed=m)
    bias = make_weight(1, n, seed=9, scale=0.5).view(-1)
    y = F.nf4_linear_fwd(x, packed, qs, bias)
    y_ref = o.bf16_round(bf16_to_f32_np(x) @ w_ref.T + bf16_to_f32_np(bias))
    assert_close_bf16(bf16_to_f32_np(y), y_ref, TOL)
    # through the module, as model.generate() would call it (no grad, one token)
    if nested and n == 4096:
        lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
        lin.weight = q.nn.Params4bit.from_prequantized(packed, qs.as_dict(packed=True), device="cuda", module=lin)
        with torch.no_grad():
            y1 = lin(x[:1].view(1, 1, k))
        assert_close_bf16(bf16_to_f32_np(y1.view(1, n)), o.bf16_round(bf16_to_f32_np(x[:1]) @ w_ref.T), TOL)


@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m", [1, 5, 8, 9, 16, 17, 31, 32])
@pytest.mark.parametrize("n,k", [(4096, 4096), (200, 192), (8, 64), (24, 320), (4096, 11008)])
def test_skinny_forward_up_to_32_tokens(q, c_oracle, m, n, k, nested):
    """Forward calls with 1..16 tokens and no LoRA operands run the warp-level skinny kernel (nf4_gemv.cu: mma.sync with the
    PRMT look-up output as B fragment, x staged through shared memory); 17..32 tokens cross over to the split-K wgmma kernel.
    Shapes include K/64 not a multiple of 4 (partial block groups, zero-filled slabs) and N = 8."""
    F = q.functional
    w = make_weight(n, k, seed=3 * n + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    x = make_act(m, k, seed=10 + m)
    bias = make_weight(1, n, seed=9, scale=0.5).view(-1)
    for b in (bias, None):
        y = F.nf4_linear_fwd(x, packed, qs, b)
        y_ref = bf16_to_f32_np(x) @ w_ref.T + (bf16_to_f32_np(b) if b is not None else 0.0)
        assert_close_bf16(bf16_to_f32_np(y), o.bf16_round(y_ref), TOL)


@pytest.mark.parametrize("m,n,k", [(2048, 5120, 5120), (1024, 22016, 8192), (4096, 4096, 4096), (2048, 13824, 5120)])
def test_other_model_shapes_vs_unfused(q, m, n, k):
    """Llama-2-13B / LLaMA-65B layer shapes (BASELINE.json configs 4-5) and a 4096-token batch: fused vs the bit-exact
    dequant kernel + cuBLAS, forward and dX, plus determinism."""
    F = q.functional
    w = make_weight(n, k, seed=n ^ k)
    packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
    wd = F.dequantize_4bit(packed, qs)
    x, dy = make_act(m, k, seed=3), make_act(m, n, seed=4)
    y = F.nf4_linear_fwd(x, packed, qs)
    assert_close_bf16(y.float().cpu().numpy(), torch.nn.functional.linear(x, wd).float().cpu().numpy(), TOL)
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    assert_close_bf16(dx.float().cpu().numpy(), (dy @ wd).float().cpu().numpy(), TOL)
    assert torch.equal(F.nf4_linear_fwd(x, packed, qs), y) and torch.equal(F.nf4_linear_bwd_dx(dy, packed, qs), dx)


def test_cuda_graph_capture_and_side_stream(q):
    """The C-ABI launches are asynchronous, allocation-free and use the caller's stream: a Linear4bit forward+backward
    (fused kernel + fused LoRA step) can be captured in a CUDA graph on a side stream and replayed on new data."""
    torch.manual_seed(0)
    base = q.nn.Linear4bit(512, 1024, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4").cuda()
    A = (torch.randn(16, 512, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    B = (torch.randn(1024, 16, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    x_static = torch.randn(700, 512, device="cuda", dtype=torch.bfloat16).requires_grad_(True)
    gy = torch.randn(700, 1024, device="cuda", dtype=torch.bfloat16)

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
            fwd_bwd()   # warm-up on the side stream (also exercises launching on a non-default stream)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = fwd_bwd()
    for seed in (1, 2):
        with torch.no_grad():
            x_static.copy_(torch.randn(700, 512, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16))
        g.replay()
        got = [t.clone() for t in outs]
        ref = [t.clone() for t in fwd_bwd()]   # eager on the same data
        for a_, b_ in zip(got, ref):
            assert torch.equal(a_, b_)


@pytest.mark.gpu
def test_smoke_entry_in_fresh_process():
    """__graft_entry__.smoke() in a fresh interpreter: its backward is the FIRST node torch's autograd worker thread ever
    runs, so the fused dX launch happens on a thread that has no CUDA context bound yet (regression: the driver-API
    tensor-map encode used to fail there with CUDA_ERROR_INVALID_CONTEXT)."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "smoke ok" in r.stdout


@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m,n,k,r,nprob", [(256, 256, 256, 64, 3), (300, 200, 192, 16, 2), (1000, 640, 128, 8, 3), (48, 384, 64, 64, 2),
                                           (2047, 512, 1024, 64, 3), (17, 128, 128, 0, 3), (700, 1032, 320, 32, 2),
                                           (9, 384, 320, 16, 3), (1, 256, 128, 64, 2), (16, 200, 192, 8, 3), (5, 128, 64, 0, 2)])
def test_grouped_launch_small_shapes_vs_oracle(q, c_oracle, m, n, k, r, nprob, nested):
    """`qb200_nf4_linear_group`: ragged token counts (not multiples of 16), feature counts that are not multiples of 256,
    one- and two-step contractions with a LoRA step after every segment, strided U, outputs written as column slices of ONE
    buffer — forward side by side and the backward contraction-sum, against the oracle.  With 16 tokens or fewer the forward is
    one skinny launch per problem (pitched outputs and U included), the backward still the wgmma kernel."""
    F = q.functional
    packs, states, w_refs = [], [], []
    for i in range(nprob):
        packed, qs = F.quantize_4bit(make_weight(n, k, seed=31 * i + n + k), compress_statistics=nested, quant_type="nf4")
        packs.append(packed.t())
        states.append(qs)
        w_refs.append(_oracle_weight(packed, qs, c_oracle))
    x = make_act(m, k, seed=1)
    us = vs = gs = as_ = None
    if r:
        u_cat = (make_act(m, nprob * r, seed=2).float() * 0.5).to(torch.bfloat16)
        us = [u_cat[:, i * r:(i + 1) * r] for i in range(nprob)]
        vs = [make_weight(n, r, seed=20 + i, scale=0.2) for i in range(nprob)]
        gs = [(make_act(m, r, seed=40 + i).float() * 0.5).to(torch.bfloat16) for i in range(nprob)]
        as_ = [make_weight(r, k, seed=50 + i, scale=0.2) for i in range(nprob)]
    out_cat = torch.full((m, nprob * n), float("nan"), device="cuda", dtype=torch.bfloat16)
    outs = [out_cat[:, i * n:(i + 1) * n] for i in range(nprob)]
    ys = F.nf4_linear_group(False, [x] * nprob, packs, states, us=us, vs=vs, outs=outs)
    for i in range(nprob):
        ref = bf16_to_f32_np(x) @ w_refs[i].T
        if r:
            ref = ref + bf16_to_f32_np(us[i]) @ bf16_to_f32_np(vs[i]).T
        assert ys[i].data_ptr() == outs[i].data_ptr()
        assert_close_bf16(bf16_to_f32_np(ys[i]), o.bf16_round(ref), TOL)
    assert not torch.isnan(out_cat.float()).any()
    dys = [make_act(m, n, seed=30 + i) for i in range(nprob)]
    dx = F.nf4_linear_group(True, dys, packs, states, us=gs, vs=as_)
    acc = np.zeros((m, k), np.float32)
    for i in range(nprob):
        acc += bf16_to_f32_np(dys[i]) @ w_refs[i]
        if r:
            acc += bf16_to_f32_np(gs[i]) @ bf16_to_f32_np(as_[i])
    assert_close_bf16(bf16_to_f32_np(dx), o.bf16_round(acc), TOL)


@pytest.mark.parametrize("m,n,k", [(2048, 512, 256), (1500, 768, 512), (1040, 256, 128)])
def test_range_schedule_units_bit_equal_across_token_counts(q, m, n, k):
    """The range schedule cuts the token axis wherever the cost model says; an output row must not depend on which unit
    (wgmma N = 16..128) computed it: rows of a short call equal the same rows of a long call bit for bit.
    (Token counts the library serves with the split-K schedule sum fp32 partials in another order: one bf16 ulp allowed.)"""
    F = q.functional
    from qlora_b200 import _lib

    lib = _lib.load()
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=9), compress_statistics=True, quant_type="nf4")
    x = make_act(m, k, seed=5)
    dy = make_act(m, n, seed=6)
    y = F.nf4_linear_fwd(x, packed, qs)
    dx = F.nf4_linear_bwd_dx(dy, packed, qs)
    assert lib.qb200_nf4_linear_workspace_size(m, n, k, 0) == 0 and lib.qb200_nf4_linear_workspace_size(m, n, k, 1) == 0
    for m2 in (m // 2 + 8, m - 16, 800, 112, 333):
        if m2 > m:
            continue
        for is_bwd, full, inp in ((0, y, x), (1, dx, dy)):
            part = (F.nf4_linear_bwd_dx if is_bwd else F.nf4_linear_fwd)(inp[:m2].contiguous(), packed, qs)
            if lib.qb200_nf4_linear_workspace_size(m2, n, k, is_bwd) == 0:
                assert torch.equal(part, full[:m2]), (m2, is_bwd)
            else:
                assert_close_bf16(bf16_to_f32_np(part), bf16_to_f32_np(full[:m2]), TOL)


def test_fused_lora_with_dropout_branch_matches_unfused(q):
    """--lora_dropout (scripts/finetune_llama2_guanaco_7b.sh:42): the LoRA branch reads x_lora = x * mask / (1-p).  Fused
    (x_lora as a second input; LoRA dX returned as x_lora's gradient) vs peft's sequence on the SAME fixed mask."""
    torch.manual_seed(0)
    base = q.nn.Linear4bit(512, 768, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4").cuda()
    A = (torch.randn(64, 512, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    B = (torch.randn(768, 64, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    x = torch.randn(3, 100, 512, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    gy = torch.randn(3, 100, 768, device="cuda", dtype=torch.bfloat16)
    mask = ((torch.rand(3, 100, 512, device="cuda") >= 0.1).float() / 0.9).to(torch.bfloat16)
    y = q.lora_linear4bit(x, base, A, B, 0.25, x_lora=x * mask)
    y.backward(gy)
    got = [y.detach().float(), x.grad.float(), A.grad.float(), B.grad.float()]
    x2, A2, B2 = (t.detach().clone().requires_grad_(True) for t in (x, A, B))
    y2 = base(x2) + torch.nn.functional.linear(torch.nn.functional.linear(x2 * mask, A2), B2) * 0.25
    y2.backward(gy)
    ref = [y2.detach().float(), x2.grad.float(), A2.grad.float(), B2.grad.float()]
    for name, a_, b_ in zip(("y", "dx", "dA", "dB"), got, ref):
        e = rel_err(a_.cpu().numpy(), b_.cpu().numpy())
        assert e <= 4e-3, (name, e)
    # the masked positions really are masked in the LoRA part of dX: with a zero base gradient path removed
    assert not torch.equal(got[1], torch.zeros_like(got[1]))


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_grouped_lora_autograd_matches_per_linear(q, dropout, dtype):
    """`lora_linear4bit_group` (q/k/v in one launch per direction, batched A projections, one dA GEMM) vs three
    `lora_linear4bit` calls: outputs, input gradient (sum over the three) and every adapter gradient."""
    torch.manual_seed(1)
    n_in, n_out, r = 512, 768, 32
    bases = [q.nn.Linear4bit(n_in, n_out, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4").cuda() for _ in range(3)]
    As = [(torch.randn(r, n_in, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True) for _ in range(3)]
    Bs = [(torch.randn(n_out, r, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True) for _ in range(3)]
    x = torch.randn(2, 150, n_in, device="cuda", dtype=dtype, requires_grad=True)
    gys = [torch.randn(2, 150, n_out, device="cuda", dtype=dtype) for _ in range(3)]
    masks = [((torch.rand(2, 150, n_in, device="cuda") >= 0.1).float() / 0.9).to(torch.bfloat16) for _ in range(3)]
    xls = [x.to(torch.bfloat16) * mk for mk in masks] if dropout else None
    ys = q.lora_linear4bit_group(x, bases, As, Bs, 0.5, xls)
    torch.autograd.backward(ys, gys)
    got = [t.detach().float() for t in ys] + [x.grad.float()] + [t.grad.float() for t in As + Bs]
    assert all(y.dtype == dtype for y in ys) and x.grad.dtype == dtype
    x2 = x.detach().clone().requires_grad_(True)
    As2 = [t.detach().clone().requires_grad_(True) for t in As]
    Bs2 = [t.detach().clone().requires_grad_(True) for t in Bs]
    ys2 = [q.lora_linear4bit(x2, bases[i], As2[i], Bs2[i], 0.5, None if not dropout else x2.to(torch.bfloat16) * masks[i]) for i in range(3)]
    torch.autograd.backward(ys2, gys)
    ref = [t.detach().float() for t in ys2] + [x2.grad.float()] + [t.grad.float() for t in As2 + Bs2]
    for idx, (a_, b_) in enumerate(zip(got, ref)):
        e = rel_err(a_.cpu().numpy(), b_.cpu().numpy())
        # the batched U projection may round differently from three separate GEMMs; the summed dX rounds once instead of 3x
        assert e <= 4e-3, (idx, e)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_two_devices_in_one_process(q, c_oracle):
    """ADVICE r1: the reference's default non-DDP path spans several GPUs from ONE process (`device_map='auto'`, qlora.py:300-304
    only pins a device under DDP).  The dynamic-shared-memory opt-in and the SM-pair count are per device: fused forward/dX
    and a grouped launch must work on cuda:1 after cuda:0 was used (and vice versa)."""
    F = q.functional
    for dev in ("cuda:0", "cuda:1", "cuda:0"):
        with torch.cuda.device(dev):
            w = make_weight(384, 512, seed=3, device=dev)
            packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
            w_ref = _oracle_weight(packed, qs, c_oracle)
            x, dy = make_act(900, 512, seed=1, device=dev), make_act(900, 384, seed=2, device=dev)   # > 768 tokens: no split-K
            y = F.nf4_linear_fwd(x, packed, qs)
            dx = F.nf4_linear_bwd_dx(dy, packed, qs)
            assert y.device == torch.device(dev)
            assert_close_bf16(bf16_to_f32_np(y), o.bf16_round(bf16_to_f32_np(x) @ w_ref.T), TOL)
            assert_close_bf16(bf16_to_f32_np(dx), o.bf16_round(bf16_to_f32_np(dy) @ w_ref), TOL)
            ys = F.nf4_linear_group(False, [x, x], [packed.t(), packed.t()], [qs, qs])
            assert torch.equal(ys[0], y) and torch.equal(ys[1], y)

@pytest.mark.parametrize("m", [1, 4])
def test_skinny_chain_right_after_quantize(q, m):
    """The skinny kernels are programmatic dependent launches that prefetch their weights before waiting for the previous
    kernel of the stream.  Weights written by the kernel just before (quantize -> forward with no sync in between) and
    activations produced by the previous skinny launch (a decode chain) must still be seen complete."""
    F = q.functional
    n = k = 2048
    x0 = make_act(m, k, seed=70)
    for it in range(6):
        w = make_weight(n, k, seed=100 + it)
        packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
        y1 = F.nf4_linear_fwd(x0, packed, qs)           # reads `packed` written one launch earlier
        y2 = F.nf4_linear_fwd(y1, packed, qs)           # reads the previous launch's output
        y3 = F.nf4_linear_fwd(y2, packed, qs)
        torch.cuda.synchronize()
        r1 = F.nf4_linear_fwd(x0, packed, qs)
        torch.cuda.synchronize()
        r2 = F.nf4_linear_fwd(r1, packed, qs)
        torch.cuda.synchronize()
        r3 = F.nf4_linear_fwd(r2, packed, qs)
        torch.cuda.synchronize()
        assert torch.equal(y1, r1) and torch.equal(y2, r2) and torch.equal(y3, r3)

@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("m,r", [(1, 64), (1, 8), (3, 16), (8, 64), (16, 64), (16, 24)])
@pytest.mark.parametrize("n,k", [(4096, 4096), (200, 192), (24, 320)])
def test_skinny_forward_with_lora_operands(q, c_oracle, m, r, n, k, nested):
    """Generation with the adapters attached (the reference's usual inference set-up: peft adds lora_B(lora_A(x)) to the bnb
    GEMV): 1..16 tokens WITH LoRA operands stay on the skinny kernels, the U . V^T term is their epilogue.  Checked against
    the oracle; a U buffer wider than r (row pitch) and a bias are covered too."""
    F = q.functional
    w = make_weight(n, k, seed=7 * n + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
    w_ref = _oracle_weight(packed, qs, c_oracle)
    x = make_act(m, k, seed=20 + m)
    u_wide = make_act(m, r + 8, seed=21 + r)
    u = u_wide[:, :r]                                     # row pitch r + 8
    v = make_weight(n, r, seed=22 + r, scale=0.05)
    bias = make_weight(1, n, seed=9, scale=0.5).view(-1)
    ws = F._lib.load().qb200_nf4_linear_workspace_size(m, n, k, 0)
    assert ws == 0                                        # no split-K workspace: not the wgmma kernel
    for b in (None, bias):
        y = F.nf4_linear_fwd_lora(x, packed, qs, u, v, b)
        y_ref = bf16_to_f32_np(x) @ w_ref.T + bf16_to_f32_np(u.contiguous()) @ bf16_to_f32_np(v).T
        if b is not None:
            y_ref = y_ref + bf16_to_f32_np(b)
        assert_close_bf16(bf16_to_f32_np(y), o.bf16_round(y_ref), TOL)
    # the module-level entry a peft-style wrapper calls
    if nested and (n, k) == (4096, 4096) and r == 64:
        lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
        lin.weight = q.nn.Params4bit.from_prequantized(packed, qs.as_dict(packed=True), device="cuda", module=lin)
        lora_a = make_weight(r, k, seed=30, scale=0.05)
        with torch.no_grad():
            y2 = q.lora.lora_linear4bit(x.view(1, m, k), lin, lora_a, v, 0.25)
        u2 = (bf16_to_f32_np(x) @ bf16_to_f32_np(lora_a).T) * 0.25
        y2_ref = bf16_to_f32_np(x) @ w_ref.T + o.bf16_round(u2) @ bf16_to_f32_np(v).T
        assert_close_bf16(bf16_to_f32_np(y2.view(m, n)), o.bf16_round(y2_ref), 2 * TOL)

@pytest.mark.parametrize("m", [1, 3, 8, 16])
@pytest.mark.parametrize("k,r", [(4096, 64), (11008, 192), (320, 8), (64, 16)])
def test_lora_project_few_tokens(q, m, k, r):
    """`qb200_lora_project`: U = scale * x . A^T for a decode step, against fp32 numpy (bf16 operands, one rounding);
    dense and pitched x, and the error for more than 16 tokens."""
    F = q.functional
    a = make_weight(r, k, seed=r + k, scale=0.05)
    x_wide = make_act(m, k + 64, seed=m + k)
    ref = None
    for x in (x_wide[:, :k].contiguous(), x_wide[:, :k]):
        u = F.lora_project(x, a, 0.25)
        assert u.shape == (m, r) and u.dtype == torch.bfloat16
        ref = o.bf16_round((bf16_to_f32_np(x.contiguous()) @ bf16_to_f32_np(a).T) * np.float32(0.25))
        assert_close_bf16(bf16_to_f32_np(u), ref, TOL)
    # the same numbers as the cuBLAS form the training path uses
    u_mm = torch.addmm(torch.empty(m, r, dtype=torch.bfloat16, device="cuda"), x_wide[:, :k].contiguous(), a.t(), beta=0.0, alpha=0.25)
    assert_close_bf16(bf16_to_f32_np(u_mm), ref, TOL)
    with pytest.raises(Exception):
        F.lora_project(make_act(17, k, seed=1), a, 1.0)

