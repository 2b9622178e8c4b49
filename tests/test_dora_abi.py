"""CPU tests of the row-scaled grouped entry point: its arguments are validated before any launch (no GPU needed)."""
import ctypes as ct


def test_scaled_group_argument_errors_do_not_need_a_gpu():
    from qlora_b200 import _lib

    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    base = ct.addressof(buf)
    p = base + (-base % 16)                                   # 16-byte aligned host address, never dereferenced
    pr = _lib.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p)
    probs = (_lib.Nf4Problem * 1)(pr)
    ok_scales = (ct.c_void_p * 1)(p)
    # a NULL row-scale array is rejected (NULL entries, not a NULL array, mean "unscaled")
    assert lib.qb200_nf4_linear_group_scaled(0, 1, ct.addressof(probs), None, 0, 8, 128, 128, 2, None, 0, None) == -1
    assert b"row-scale array" in lib.qb200_last_error()
    # a row scale must be 4-byte aligned fp32
    bad = (ct.c_void_p * 1)(p + 2)
    assert lib.qb200_nf4_linear_group_scaled(0, 1, ct.addressof(probs), ct.addressof(bad), 0, 8, 128, 128, 2, None, 0, None) == -1
    assert b"4-byte aligned" in lib.qb200_last_error()
    # the checks of qb200_nf4_linear_group apply unchanged
    assert lib.qb200_nf4_linear_group_scaled(0, 4, ct.addressof(probs), ct.addressof(ok_scales), 0, 8, 128, 128, 2, None, 0, None) == -1
    assert lib.qb200_nf4_linear_group_scaled(0, 1, ct.addressof(probs), ct.addressof(ok_scales), 0, 8, 128, 96, 2, None, 0, None) == -2
    assert b"multiple of 64" in lib.qb200_last_error()
    assert lib.qb200_nf4_linear_group_scaled(0, 1, ct.addressof(probs), ct.addressof(ok_scales), 12, 8, 128, 128, 2, None, 0, None) == -2
    assert lib.qb200_nf4_linear_group_scaled(1, 1, ct.addressof(probs), ct.addressof(ok_scales), 0, 8, 128, 128, 7, None, 0, None) == -1
    nb = _lib.Nf4Problem(inp=p, packed=p, out=p)              # no absmax at all
    probs_nb = (_lib.Nf4Problem * 1)(nb)
    assert lib.qb200_nf4_linear_group_scaled(0, 1, ct.addressof(probs_nb), ct.addressof(ok_scales), 0, 8, 128, 128, 2, None, 0, None) == -1
