"""The scratch kernel's output epilogue (nf4_gemm_wgmma.cuh, namespace sc): each consumer warpgroup stages its bf16 results
in shared memory and TMA-stores them in 16-token boxes that cover exactly its unit's tokens.  The stores must land where the
register epilogue put them: bitwise the fused kernel's outputs at token counts whose units end off 256- and off 32-token
boundaries, nothing outside the call's [T, F] output of a caller-pitched buffer, and outputs whose base or pitch TMA cannot
address (not 16-byte aligned) run the fused kernel instead."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_helpers import make_act, make_weight

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_case(path, **env):
    env = dict(os.environ, QB200_SPLITK_MAX_T="0", **env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "scratch_epilogue_case.py"), str(path)],
                       capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(path)


@pytest.fixture(scope="module")
def fused_outputs(tmp_path_factory):
    return _run_case(tmp_path_factory.mktemp("fused") / "fused.npz", QB200_SCRATCH_MIN_M=str(1 << 30))


@pytest.mark.gpu
@pytest.mark.parametrize("reserved", ["0", "100"])
def test_scratch_epilogue_matches_fused_kernel_bitwise(tmp_path, fused_outputs, reserved):
    """Grouped q/k/v and gate/up, forward (LoRA + bias, and fp32 output) and dX (LoRA), at 1552, 1808, 2000 and 3000 tokens;
    reserved = 100 leaves 32 CTAs on an H100 SXM, which cuts the tails elsewhere."""
    a = _run_case(tmp_path / "scratch.npz", QB200_SCRATCH_MIN_M="1536", QB200_RESERVED_SMS=reserved)
    b = fused_outputs
    assert sorted(a.files) == sorted(b.files) and len(a.files) == 4 * ((3 + 3 + 1) + (2 + 2 + 1))
    diff = [name for name in a.files if not np.array_equal(a[name], b[name])]
    assert not diff, diff


def _problem(m, n, k, seed):
    import qlora_b200.functional as F

    packed, qs = F.quantize_4bit(make_weight(n, k, seed=seed), compress_statistics=True, quant_type="nf4")
    return F, packed.t(), qs, make_act(m, k, seed=seed + 1), make_weight(1, n, seed=seed + 2).view(-1)


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.gpu
def test_scratch_epilogue_writes_only_the_output(tmp_path):
    """A caller-pitched output: rows >= T and columns >= F of the [T + 64, ld_out] buffer keep their sentinel."""
    m, n, k, ld = 2000, 4096 + 8, 4096, 4096 + 72
    F, packed, qs, x, bias = _problem(m, n, k, 210)
    sentinel = torch.tensor(-12345.0, dtype=torch.bfloat16)
    buf = torch.full((m + 64, ld), sentinel.item(), dtype=torch.bfloat16, device="cuda")
    y = F.nf4_linear_group(False, [x], [packed], [qs], biases=[bias], outs=[buf[:m, :n]])[0]
    assert y.data_ptr() == buf.data_ptr()
    ref = F.nf4_linear_fwd(x, packed, qs, bias)
    torch.cuda.synchronize()
    assert torch.equal(buf[:m, :n], ref)
    assert bool((buf[:m, n:] == sentinel.item()).all()) and bool((buf[m:] == sentinel.item()).all())


@pytest.mark.gpu
@pytest.mark.parametrize("offset,ld_pad", [(1, 0), (0, 4)], ids=["base", "pitch"])
def test_unaligned_output_takes_the_fused_kernel(offset, ld_pad):
    """An output whose base (2 bytes off) or pitch (F + 4 elements) is not 16-byte aligned runs the fused kernel, with the
    same bits as the scratch path's aligned output."""
    m, n, k = 2048, 4096, 4096
    F, packed, qs, x, bias = _problem(m, n, k, 220)
    ref = F.nf4_linear_fwd(x, packed, qs, bias)
    ld = n + ld_pad
    buf = torch.zeros(offset + m * ld, dtype=torch.bfloat16, device="cuda")
    out = buf[offset:].view(m, ld)[:, :n]
    assert out.data_ptr() % 16 != 0 or (out.stride(0) * 2) % 16 != 0
    names = _kernel_names(lambda: F.nf4_linear_group(False, [x], [packed], [qs], biases=[bias], outs=[out]))
    assert any("nf4_gemm_wgmma_kernel" in s for s in names) and not any("scratch_gemm" in s for s in names), names
    assert torch.equal(out, ref)
    names = _kernel_names(lambda: F.nf4_linear_fwd(x, packed, qs, bias))
    assert any("scratch_gemm" in s for s in names), names
