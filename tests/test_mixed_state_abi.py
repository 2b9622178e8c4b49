"""CPU tests of `qb200_nf4_linear_group_ex`: the (dtype, state_dtype, out_dtype) combinations it accepts, and QB200_EINVAL for
every other one before any launch (no GPU needed)."""
import ctypes as ct
import itertools

from qlora_b200 import _lib

F32, F16, BF16 = 0, 1, 2
SUPPORTED = {(BF16, s, o) for s in (BF16, F16, F32) for o in (BF16, F32, F16)} | {(F16, s, o) for s in (F16, F32) for o in (F16, F32)}


def _aligned(buf):
    base = ct.addressof(buf)
    return base + (-base % 16)                                 # 16-byte aligned host address, never dereferenced


def _ex(lib, probs, dtype, state_dtype, out_dtype, k=128):
    return lib.qb200_nf4_linear_group_ex(0, dtype, state_dtype, 1, probs, 0, 8, 128, k, out_dtype, None, 0, None)


def test_ex_rejects_every_unsupported_dtype_combination_before_any_launch():
    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    p = _aligned(buf)
    probs = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p))
    codes = (F32, F16, BF16, 3, -1)
    rejected = 0
    for combo in itertools.product(codes, repeat=3):
        if combo in SUPPORTED:
            continue
        assert _ex(lib, ct.addressof(probs), *combo) == -1, combo
        assert b"unsupported (dtype, state_dtype, out_dtype)" in lib.qb200_last_error(), combo
        # the dtype check comes first: a null problem array does not change the answer
        assert _ex(lib, None, *combo) == -1 and b"unsupported (dtype" in lib.qb200_last_error(), combo
        rejected += 1
    assert rejected == 5 ** 3 - len(SUPPORTED)
    # the one pair kept off the fused path on purpose: fp16 compute over a bf16 state
    assert _ex(lib, ct.addressof(probs), F16, BF16, F16) == -1


def test_ex_accepts_the_supported_combinations_up_to_the_shape_check():
    """Every supported combination passes the dtype check and stops at the shape check (K % 64 != 0), which also returns
    before any launch."""
    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    p = _aligned(buf)
    probs = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p))
    for combo in sorted(SUPPORTED):
        assert _ex(lib, ct.addressof(probs), *combo, k=96) == -2, combo
        assert b"multiple of 64" in lib.qb200_last_error(), combo
    # argument checks of the other grouped forms apply unchanged
    assert _ex(lib, None, BF16, F16, F16) == -1 and b"1..3 problems" in lib.qb200_last_error()
    bad = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(inp=p, packed=p, out=p))          # no absmax at all
    assert _ex(lib, ct.addressof(bad), BF16, F16, F16) == -1
