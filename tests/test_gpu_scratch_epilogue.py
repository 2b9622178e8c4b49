"""The scratch kernel's output epilogue (nf4_gemm_wgmma.cuh, namespace sc): each consumer warpgroup stages its bf16 results
in shared memory and TMA-stores them in 16-token boxes that cover exactly its unit's tokens.  The stores must land where the
register epilogue put them: bitwise the fused kernel's outputs at token counts whose units end off 256- and off 32-token
boundaries, nothing outside the call's [T, F] outputs of a caller-pitched buffer (also through the fp32 register epilogue,
for dX, and for grouped outputs side by side), and outputs whose base or pitch TMA cannot
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
def test_scratch_epilogue_writes_only_the_output():
    """Caller-pitched outputs at partial last feature blocks (8, 120 and 64 features wide) and ragged token counts: forward
    and dX, bf16 (TMA epilogue) and fp32 (register epilogue) outputs, and a grouped forward.  Each [T, F] output is a view of
    a [T + 64, ld_out] buffer; the grouped forward's outputs sit side by side with 8 sentinel columns after each (every slice
    base stays 16-byte aligned).  Every output equals the unpitched call's, and every element outside them keeps its
    sentinel."""
    import qlora_b200.functional as F

    cases = [(False, torch.bfloat16, 1), (False, torch.float32, 1), (True, torch.bfloat16, 1), (True, torch.float32, 1),
             (False, torch.bfloat16, 3)]
    for m, n, k in [(2000, 4104, 4160), (3000, 11000, 1088), (1543, 200, 192)]:
        ps, qss, biases = [], [], []
        for i in range(3):
            _, packed, qs, x, bias = _problem(m, n, k, 210 + 3 * i)
            ps.append(packed)
            qss.append(qs)
            biases.append(bias)
        dy = make_act(m, n, seed=209)
        for is_bwd, out_dtype, nprob in cases:
            what = (m, n, k, "dx" if is_bwd else "fwd", out_dtype, nprob)
            f_out = k if is_bwd else n
            assert F._lib.load().qb200_nf4_linear_scratch_size(nprob, m, n, k, int(is_bwd)) == nprob * n * k * 2, what
            pitch = f_out + 8
            ld = nprob * pitch + 64
            sentinel = torch.tensor(-12345.0, dtype=out_dtype).item()
            buf = torch.full((m + 64, ld), sentinel, dtype=out_dtype, device="cuda")
            outs = [buf[:m, i * pitch:i * pitch + f_out] for i in range(nprob)]
            if is_bwd:
                refs = [F.nf4_linear_bwd_dx(dy, ps[0], qss[0], out_dtype=out_dtype)]   # unpitched
                ys = [F.nf4_linear_group(True, [dy], ps[:1], qss[:1], outs=outs, out_dtype=out_dtype)]
            else:
                refs = F.nf4_linear_group(False, [x] * nprob, ps[:nprob], qss[:nprob], biases=biases[:nprob], out_dtype=out_dtype)
                ys = F.nf4_linear_group(False, [x] * nprob, ps[:nprob], qss[:nprob], biases=biases[:nprob], outs=outs,
                                        out_dtype=out_dtype)
            torch.cuda.synchronize()
            inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
            for i, (y, ref) in enumerate(zip(ys, refs)):
                assert y.data_ptr() == outs[i].data_ptr(), what
                assert torch.equal(y, ref), (what, i)
                inside[:m, i * pitch:i * pitch + f_out] = True
            assert bool((buf[~inside] == sentinel).all()), what


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
