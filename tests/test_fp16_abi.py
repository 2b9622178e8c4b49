"""CPU tests of the typed (bf16 / fp16) entry points: dtype, out_dtype and pointer arguments are validated before any launch
(no GPU needed)."""
import ctypes as ct

from qlora_b200 import _lib

F32, F16, BF16 = 0, 1, 2


def _aligned(buf):
    base = ct.addressof(buf)
    return base + (-base % 16)                                 # 16-byte aligned host address, never dereferenced


def _group(lib, probs, dtype, out_dtype, is_bwd=0, scales=None, r=0, m=8, n=128, k=128):
    return lib.qb200_nf4_linear_group_typed(is_bwd, dtype, 1, ct.addressof(probs), scales, r, m, n, k, out_dtype, None, 0, None)


def test_typed_group_rejects_bad_dtypes_before_any_launch():
    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    p = _aligned(buf)
    probs = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p))
    for dtype in (F32, 3, -1, 7):
        assert _group(lib, probs, dtype, F32) == -1
        assert b"dtype must be 2 (bf16) or 1 (fp16)" in lib.qb200_last_error()
    # out_dtype must be the operand dtype or fp32
    assert _group(lib, probs, F16, BF16) == -1
    assert b"out_dtype must be 1 (fp16) or 0 (fp32)" in lib.qb200_last_error()
    assert _group(lib, probs, BF16, F16) == -1
    assert b"out_dtype must be 2 (bf16) or 0 (fp32)" in lib.qb200_last_error()
    assert _group(lib, probs, F16, 5) == -1


def test_typed_group_rejects_null_pointers_before_any_launch():
    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    p = _aligned(buf)
    assert lib.qb200_nf4_linear_group_typed(0, F16, 1, None, None, 0, 8, 128, 128, F16, None, 0, None) == -1
    for missing in ("inp", "packed", "out"):
        fields = dict(inp=p, packed=p, absmax_f32=p, out=p)
        fields[missing] = None
        probs = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(**fields))
        for out_dtype in (F16, F32):
            assert _group(lib, probs, F16, out_dtype) == -1
            assert b"null pointer" in lib.qb200_last_error()
    probs = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(inp=p, packed=p, out=p))     # no absmax at all
    assert _group(lib, probs, F16, F16) == -1
    probs = (_lib.Nf4Problem * 1)(_lib.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p))
    assert _group(lib, probs, F16, F16, r=16) == -1                          # LoRA rank without U / V
    assert b"null LoRA operand" in lib.qb200_last_error()
    # the shape checks of the bf16 form apply unchanged
    assert _group(lib, probs, F16, F16, k=96) == -2
    assert b"multiple of 64" in lib.qb200_last_error()
    bad = (ct.c_void_p * 1)(p + 2)
    assert _group(lib, probs, F16, F16, scales=ct.addressof(bad)) == -1
    assert b"4-byte aligned" in lib.qb200_last_error()


def test_typed_lora_project_rejects_bad_arguments_before_any_launch():
    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    p = _aligned(buf)
    for dtype in (F32, 3):
        assert lib.qb200_lora_project_typed(dtype, p, 0, p, 1.0, p, 0, 1, 64, 8, None) == -1
        assert b"dtype must be 2 (bf16) or 1 (fp16)" in lib.qb200_last_error()
    for x, a, u in ((None, p, p), (p, None, p), (p, p, None)):
        assert lib.qb200_lora_project_typed(F16, x, 0, a, 1.0, u, 0, 1, 64, 8, None) == -1
        assert b"null pointer" in lib.qb200_last_error()
    assert lib.qb200_lora_project_typed(F16, p, 0, p, 1.0, p, 0, 17, 64, 8, None) == -2
    assert lib.qb200_lora_project_typed(F16, p + 2, 0, p, 1.0, p, 0, 1, 64, 8, None) == -1
    assert b"16-byte aligned" in lib.qb200_last_error()
