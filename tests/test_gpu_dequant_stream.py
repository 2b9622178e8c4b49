"""The table dequantize kernel (dequantize_nf4_tab_kernel) at the edges of its work partition: a warp expands runs of 32
16-byte vectors (32 values each) through a shared-memory stage, two runs per iteration, over a grid capped at 8 CTAs of 8
warps per SM.  Every output is compared bit for bit with the C oracle, and a sentinel fill around the output shows that
nothing outside [out, out + n) is written."""
import numpy as np
import pytest
import torch

import oracle_c as oc
from gpu_helpers import state_to_numpy

pytestmark = pytest.mark.gpu

SENTINEL = 0x7E7E   # a 16-bit pattern no NF4 product of the test weights takes
PAD = 64            # elements of sentinel on each side of the output (128 bytes)


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    assert torch.cuda.is_available(), "GPU tests need a GPU"
    from qlora_b200 import _lib

    _lib.load()
    return F


def grid_vectors():
    """Vectors one iteration of the capped grid covers: SMs x 8 CTAs x 8 warps x 2 runs x 32 vectors."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 8 * 2 * 32


def oracle_bits(c_oracle, packed, qs, n, dtype):
    """The oracle's fp32 product LUT[j] * absmax rounded to `dtype` (round to nearest even), as 16-bit patterns."""
    st = state_to_numpy(packed, qs)
    if st["nested"]:
        absmax = oc.nested_absmax(c_oracle, st["code256"], st["absmax_u8"], st["absmax2"], st["offset"], qs.state2.blocksize)
    else:
        absmax = st["absmax"]
    w = oc.dequantize_nf4_f32(c_oracle, st["packed"], absmax, n, qs.blocksize)
    if dtype == torch.float16:
        return w.astype(np.float16).view(np.uint16)
    b = w.view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def dequant_into_padded(F, packed, qs, n, dtype, pad):
    """dequantize_4bit into elements [pad, pad + n) of a sentinel-filled buffer; returns the whole buffer's bits."""
    buf = torch.full((n + 2 * PAD,), SENTINEL, dtype=torch.int16, device="cuda").view(dtype)
    qs.dtype = dtype
    F.dequantize_4bit(packed, qs, out=buf[pad:pad + n])
    torch.cuda.synchronize()
    return buf.view(torch.int16).cpu().numpy().view(np.uint16)


def check(F, c_oracle, nvec, bs, nested, dtype, pad=PAD, seed=0):
    n = 32 * nvec
    g = torch.Generator(device="cpu").manual_seed(seed + nvec)
    w = (torch.randn(n, generator=g) * 0.02).to(torch.bfloat16).cuda()
    packed, qs = F.quantize_4bit(w, blocksize=bs, compress_statistics=nested, quant_type="nf4")
    got = dequant_into_padded(F, packed, qs, n, dtype, pad)
    ref = oracle_bits(c_oracle, packed, qs, n, dtype)
    assert np.array_equal(got[pad:pad + n], ref), f"nvec={nvec}: {np.count_nonzero(got[pad:pad + n] != ref)} values differ"
    assert np.all(got[:pad] == SENTINEL) and np.all(got[pad + n:] == SENTINEL), "write outside the output"
    return got[pad:pad + n]


# runs of 32 vectors, a warp's two runs (64), a CTA's 512 vectors: one short of and one past each
SMALL_NVEC = [1, 2, 31, 33, 63, 65, 511, 513, 1000]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("nested", [True, False], ids=["nested", "plain"])
@pytest.mark.parametrize("bs", [64, 256, 4096])
@pytest.mark.parametrize("nvec", SMALL_NVEC)
def test_partial_runs_bit_exact(F, c_oracle, nvec, bs, nested, dtype):
    check(F, c_oracle, nvec, bs, nested, dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("nested", [True, False], ids=["nested", "plain"])
@pytest.mark.parametrize("extra", [-1, 1, 33, None])
def test_grid_stride_bit_exact(F, c_oracle, extra, nested, dtype):
    """One vector short of and one past the capped grid's span, a partial run in the second iteration, and a span
    and a half (the last iteration leaves whole warps without work)."""
    span = grid_vectors()
    nvec = 3 * span // 2 if extra is None else (span + extra if extra != 33 else 2 * span + 33)
    check(F, c_oracle, nvec, 64, nested, dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("nested", [True, False], ids=["nested", "plain"])
@pytest.mark.parametrize("shape", [(4096, 4096), (11008, 4096)])
def test_7b_shapes_bit_exact(F, c_oracle, shape, nested, dtype):
    check(F, c_oracle, shape[0] * shape[1] // 32, 64, nested, dtype)


@pytest.mark.parametrize("nested", [True, False], ids=["nested", "plain"])
def test_16_byte_aligned_output_same_bits(F, c_oracle, nested):
    """The table kernel takes 32-byte aligned outputs; a 16-byte aligned one takes the fallback kernel, with the same bits."""
    nvec = 1000
    a = check(F, c_oracle, nvec, 64, nested, torch.bfloat16, pad=PAD)          # 128-byte offset: table kernel
    b = check(F, c_oracle, nvec, 64, nested, torch.bfloat16, pad=PAD - 8)      # 112 bytes: 16-byte aligned only
    assert np.array_equal(a, b)
