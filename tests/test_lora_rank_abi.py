"""LoRA ranks of the NF4 linear entry points, without a GPU: multiples of 8 in [8, 256] pass the rank check of every entry
point that takes a rank, every other nonzero rank returns QB200_EUNSUPPORTED before any launch, and the Python gate that
picks the fused LoRA path agrees."""
import ctypes as ct
import types

import pytest
import torch

EUNSUPPORTED, EINVAL = -2, -1
BAD_RANKS = [264, 68, 4, 512, -8]
GOOD_RANKS = [8, 64, 72, 128, 136, 200, 256]


@pytest.fixture(scope="module")
def env():
    from qlora_b200 import _lib

    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    base = ct.addressof(buf)
    p = base + (-base % 16)                                   # 16-byte aligned host address, never dereferenced
    return lib, _lib, buf, p


def _calls(env, R, with_lora_operands):
    """(name, thunk) for every entry point that takes a LoRA rank: a forward of 8 tokens over a 128 x 128 plain state."""
    lib, L, _, p = env
    u = p if with_lora_operands else None
    pr = L.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p, U=u, V=u)
    probs = (L.Nf4Problem * 1)(pr)
    pp = ct.addressof(probs)
    scales = (ct.c_void_p * 1)(None)
    flag = ct.c_int(0)
    m, n, k = 8, 128, 128
    return [
        ("fwd_lora", lambda: lib.qb200_nf4_linear_fwd_lora(p, p, None, None, None, None, p, None, u, u, R, p, m, n, k, None)),
        ("bwd_dx_lora", lambda: lib.qb200_nf4_linear_bwd_dx_lora(p, p, None, None, None, None, p, u, u, R, p, m, n, k, None)),
        ("ex", lambda: lib.qb200_nf4_linear_ex(0, p, p, None, None, None, None, p, None, u, u, R, p, m, n, k, None, 0, None)),
        ("group", lambda: lib.qb200_nf4_linear_group(0, 1, pp, R, m, n, k, 2, None, 0, None)),
        ("group_scaled", lambda: lib.qb200_nf4_linear_group_scaled(0, 1, pp, ct.addressof(scales), R, m, n, k, 2, None, 0, None)),
        ("group_typed", lambda: lib.qb200_nf4_linear_group_typed(1, 1, 1, pp, None, R, m, n, k, 1, None, 0, None)),
        ("group_ex", lambda: lib.qb200_nf4_linear_group_ex(0, 2, 1, 1, pp, R, m, n, k, 2, None, 0, None)),
        ("group_reuse", lambda: lib.qb200_nf4_linear_group_reuse(0, 2, 2, 1, pp, R, m, n, k, 2, None, 0, ct.byref(flag), None)),
    ]


@pytest.mark.parametrize("R", BAD_RANKS)
def test_unsupported_ranks_are_refused_before_any_launch(env, R):
    lib = env[0]
    for name, call in _calls(env, R, with_lora_operands=True):
        assert call() == EUNSUPPORTED, name
        assert b"multiple of 8 in [8, 256]" in lib.qb200_last_error(), name


@pytest.mark.parametrize("R", GOOD_RANKS)
def test_supported_ranks_pass_the_rank_check(env, R):
    """With the LoRA operands left NULL the call fails on them, after the rank check, and still before any launch."""
    lib = env[0]
    for name, call in _calls(env, R, with_lora_operands=False):
        assert call() == EINVAL, name
        assert b"null LoRA operand" in lib.qb200_last_error(), name


def _state(nested=False, dtype=torch.bfloat16):
    return types.SimpleNamespace(quant_type="nf4", blocksize=64, shape=torch.Size([4096, 4096]), dtype=dtype, nested=nested,
                                 state2=types.SimpleNamespace(blocksize=256))


def test_python_gate_follows_the_library():
    import qlora_b200.functional as F

    for cdt, sdt in ((torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16)):
        qs = _state(dtype=sdt)
        for r in GOOD_RANKS:
            assert F.lora_fused_supported(qs, cdt, r), (cdt, r)
        for r in (264, 132, 68, 4, 0, 512):
            assert not F.lora_fused_supported(qs, cdt, r), (cdt, r)
