"""`bitsandbytes.matmul_4bit` / `MatMul4Bit` on the fused H100 kernel.

Reference semantics being honoured (upstream bitsandbytes/autograd/_functions.py, reached from
qlora.py:249 via `bnb.nn.Linear4bit.forward`; SURVEY.md 8a rows a8, a11):

    forward : out = F.linear(A, dequantize_4bit(B, state).to(A.dtype).t(), bias)
    backward: grad_A = grad_out @ dequantize_4bit(B, state).to(grad_out.dtype).t()   (B is weight.t())
              grad_B = None (frozen base weight: no dW GEMM), grad_bias = grad_out.sum(0)

Here forward and dX run as ONE hand-written sm_90a kernel each (NF4 nibbles -> 16-bit tiles in
shared memory -> wgmma), so the dequantized W never reaches HBM.  The fused compute dtypes are
bf16 (over a bf16, fp16 or fp32 quant state) and fp16 (over an fp16 or fp32 quant state: `qlora.py --fp16`,
`bnb_4bit_compute_dtype=torch.float16`); for those, the kernels' weights are exactly
`dequantize_4bit(B, state).to(compute_dtype)`: fp16_rn / bf16_rn(LUT[j]*absmax), and bf16_rn(fp16_rn(LUT[j]*absmax)) for an
fp16 state under bf16 compute.  Inputs the fused kernel does not cover (fp32 compute dtype, a bf16 state under fp16
compute, K % 64 != 0, ...) take the unfused *GPU* path (our dequant kernel + cuBLAS), which is also the
"bnb-equivalent" baseline timed in bench.py.
"""
from __future__ import annotations

import warnings
from math import prod
from typing import Optional

import torch

from . import functional as F

# Set to False to force the unfused (dequantize -> cuBLAS) GPU path, e.g. for A/B timing.
USE_FUSED = True


def _unfused_weight(B: torch.Tensor, state: F.QuantState, dtype: torch.dtype) -> torch.Tensor:
    # B is the [1, n/2] transposed view -> dequantize_4bit returns W^T [K, N]
    return F.dequantize_4bit(B, state).to(dtype)


class MatMul4Bit(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A, B, out=None, bias=None, quant_state: Optional[F.QuantState] = None, compute_dtype=None):
        # `compute_dtype` (extension): Linear4bit.forward's `x.to(compute_dtype)` ... `.to(inp_dtype)` folded into this node —
        # fp32 activations (bf16 or fp16 compute) and fp16 activations (bf16 compute) are cast to the compute dtype once, and
        # the kernel epilogue writes the rounded result in the input's dtype (forward) / the input gradient (backward): the
        # two output-side cast passes of a7 disappear.
        ctx.io_dtype = None
        if compute_dtype is not None and A.dtype != compute_dtype:
            foldable = ((A.dtype == torch.float32 and compute_dtype in (torch.bfloat16, torch.float16))
                        or (A.dtype == torch.float16 and compute_dtype == torch.bfloat16))
            if (foldable and USE_FUSED and out is None and prod(A.shape) > 0 and B.shape[0] == 1
                    and F.fused_supported(quant_state, compute_dtype)):
                ctx.io_dtype = A.dtype
            else:  # not coverable by the epilogue: behave exactly like the module-side casts
                raise RuntimeError("MatMul4Bit: compute_dtype folding needs fp32 input + bf16/fp16 compute or fp16 input + bf16 "
                                   "compute, on the fused path")
        ctx.is_empty = False
        if prod(A.shape) == 0:
            ctx.is_empty = True
            ctx.A = A
            ctx.B = B
            ctx.bias = bias
            B_shape = quant_state.shape
            if A.shape[-1] == B_shape[0]:
                return torch.empty(A.shape[:-1] + B_shape[1:], dtype=A.dtype, device=A.device)
            return torch.empty(A.shape[:-1] + B_shape[:1], dtype=A.dtype, device=A.device)

        fused = ctx.io_dtype is not None or (USE_FUSED and B.shape[0] == 1 and F.fused_supported(quant_state, A.dtype))
        cdt = compute_dtype if ctx.io_dtype is not None else A.dtype
        scratch = None
        if fused:
            b = bias if (bias is None or bias.dtype == cdt) else bias.to(cdt)
            ys, scratch = F.nf4_linear_group(False, [F.as_compute_2d(A, cdt)], [B], [quant_state], None if b is None else [b],
                                             out_dtype=F.out_dtype_for(A.dtype, cdt), return_scratch=True)
            output = ys[0].view(*A.shape[:-1], quant_state.shape[0])
        else:
            output = torch.nn.functional.linear(A, _unfused_weight(B, quant_state, A.dtype).t(), bias)
        kept = F.scratch_to_save(scratch, ctx.needs_input_grad[0])   # a checkpoint recompute's W copy, for the dX launch
        # only the PACKED weight is kept for backward (no bf16 W is saved)
        ctx.save_for_backward(*([B] if any(ctx.needs_input_grad[:2]) else []), *kept)
        ctx.kept_scratch = bool(kept)
        if out is not None:
            out.copy_(output)
            output = out

        ctx.state = quant_state
        ctx.fused, ctx.cdt = fused, cdt
        ctx.dtype_A, ctx.dtype_B, ctx.dtype_bias = A.dtype, B.dtype, None if bias is None else bias.dtype
        return output

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.is_empty:
            bias_grad = None if ctx.bias is None else torch.zeros_like(ctx.bias)
            return torch.zeros_like(ctx.A), torch.zeros_like(ctx.B), None, bias_grad, None, None
        req_gradA, _, _, req_gradBias = ctx.needs_input_grad[:4]
        grad_A, grad_B, grad_bias = None, None, None
        if req_gradBias:
            # sum over every leading dim (upstream sums dim 0 only, which is wrong for 3-D inputs)
            grad_bias = grad_output.reshape(-1, grad_output.shape[-1]).sum(0, dtype=ctx.dtype_bias)
        if req_gradA:
            saved = ctx.saved_tensors
            B = saved[0]
            if ctx.fused and (ctx.io_dtype is not None or grad_output.dtype == ctx.cdt):
                scratch = F.saved_scratch(saved) if ctx.kept_scratch else None
                dx = F.nf4_linear_group(True, [F.as_compute_2d(grad_output, ctx.cdt)], [B], [ctx.state],
                                        out_dtype=F.out_dtype_for(ctx.dtype_A, ctx.cdt), w_scratch=scratch)
                grad_A = dx.view(*grad_output.shape[:-1], ctx.state.shape[1])
            else:
                grad_A = torch.matmul(grad_output, _unfused_weight(B, ctx.state, grad_output.dtype).t())
        return grad_A, grad_B, None, grad_bias, None, None


def matmul_4bit(A: torch.Tensor, B: torch.Tensor, quant_state: F.QuantState, out: Optional[torch.Tensor] = None,
                bias: Optional[torch.Tensor] = None, compute_dtype: Optional[torch.dtype] = None):
    """`bnb.matmul_4bit(A, B=weight.t(), quant_state=..., bias=...)`.

    Upstream diverts single-token, no-grad calls to a GEMV kernel (SURVEY.md 8f-2); here every forward with at most
    16 tokens and no LoRA operands is dispatched inside the C library to the skinny kernel (nf4_gemv.cu).
    """
    assert quant_state is not None
    if not A.is_cuda:
        raise RuntimeError("qlora_b200.matmul_4bit: CUDA tensors only (no CPU fallback)")
    return MatMul4Bit.apply(A, B, out, bias, quant_state, compute_dtype)
