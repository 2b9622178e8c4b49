"""The segmented mixed-adapter entry points without a GPU: they are declared and exported, the workspace size depends only on
(M, n_adapters), their argument errors come back before any launch, the custom op is registered, and the names form picks
its branch on the host."""
import ctypes as ct
import os
import re

import pytest

EUNSUPPORTED, EINVAL = -2, -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("qb200_lora_segment_table", "qb200_lora_shrink_segmented", "qb200_lora_expand_segmented")


@pytest.fixture(scope="module")
def env():
    from qlora_b200 import _lib

    lib = _lib.load()
    buf = (ct.c_char * 4096)()
    base = ct.addressof(buf)
    p = base + (-base % 16)                                   # 16-byte aligned host address, never dereferenced
    return lib, _lib, buf, p


def test_exports_are_declared_and_bound(env):
    lib, L, _, _ = env
    header = open(os.path.join(ROOT, "include", "qlora_b200.h")).read()
    for name in NAMES:
        assert re.search(r"\bint " + name + r"\(", header), name
        assert name in L.EXPORTED_SYMBOLS and getattr(lib, name) is not None
    assert re.search(r"\bint64_t qb200_lora_segment_workspace_size\(", header)


def test_workspace_size(env):
    lib = env[0]
    size = lib.qb200_lora_segment_workspace_size
    assert size(0, 4) == 0 and size(17, 0) == 0 and size(-1, 4) == 0
    # perm [M], offsets [n + 2], tiles [ceil(M / 64) + n] of 16 bytes, counts and tile offsets [2 (n + 1)], each 16-aligned
    for m, n in ((17, 1), (300, 16), (1600, 1000), (1 << 20, 7)):
        pad = lambda b: (b + 15) // 16 * 16  # noqa: E731
        assert size(m, n) == pad(4 * m) + pad(4 * (n + 2)) + 16 * ((m + 63) // 64 + n) + pad(8 * (n + 1)), (m, n)
        assert size(m, n) % 16 == 0


def _table(env, **kw):
    lib, _, _, p = env
    a = dict(rows=p, M=300, n=16, ws=p, ws_bytes=1 << 20)
    a.update(kw)
    return lib.qb200_lora_segment_table(a["rows"], a["M"], a["n"], a["ws"], a["ws_bytes"], None)


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(rows=None), EINVAL, b"null pointer"),
    (dict(ws=None), EINVAL, b"null pointer"),
    (dict(n=0), EINVAL, b"n_adapters"),
    (dict(M=0), EINVAL, b"bad shape"),
    (dict(ws_bytes=64), EINVAL, b"workspace smaller"),
    (dict(rows="p+2"), EINVAL, b"aligned"),
    (dict(ws="p+4"), EINVAL, b"aligned"),
])
def test_segment_table_argument_errors(env, kw, rc, msg):
    p = env[3]
    kw = {k: (p + int(v[2:]) if isinstance(v, str) else v) for k, v in kw.items()}
    assert _table(env, **kw) == rc
    assert msg in env[0].qb200_last_error()


def _arrays(p, nprob):
    return (ct.c_void_p * max(3, nprob))(*([p] * nprob + [None] * (3 - nprob)))


def _shrink(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, x=p, ld_x=0, tables=_arrays(p, nprob), U=_arrays(p, nprob), ld_u=0, n=16, ws=p, ws_bytes=1 << 20, M=300,
             K=4096, R=64)
    a.update(kw)
    return lib.qb200_lora_shrink_segmented(a["dtype"], nprob, a["x"], a["ld_x"], a["tables"], a["U"], a["ld_u"], a["n"], a["ws"],
                                           a["ws_bytes"], a["M"], a["K"], a["R"], None)


def _expand(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, tables=_arrays(p, nprob), U=_arrays(p, nprob), ld_u=0, out=_arrays(p, nprob), ld_out=0, n=16, ws=p,
             ws_bytes=1 << 20, M=300, N=4096, R=64)
    a.update(kw)
    return lib.qb200_lora_expand_segmented(a["dtype"], nprob, a["tables"], a["U"], a["ld_u"], a["out"], a["ld_out"], a["n"],
                                           a["ws"], a["ws_bytes"], a["M"], a["N"], a["R"], None)


COMMON = [
    (dict(dtype=0), EINVAL, b"dtype"),
    (dict(tables=None), EINVAL, b"no null pointer"),
    (dict(ws=None), EINVAL, b"no null pointer"),
    (dict(n=0), EINVAL, b"n_adapters"),
    (dict(R=4), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(R=264), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(M=0), EINVAL, b"bad shape"),
    (dict(ws_bytes=256), EINVAL, b"workspace"),
]


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(K=100), EINVAL, b"bad shape"),
    (dict(ld_x=100), EINVAL, b"row pitch"),
    (dict(ld_u=32), EINVAL, b"row pitch"),
])
def test_shrink_argument_errors(env, kw, rc, msg):
    assert _shrink(env, **kw) == rc
    assert msg in env[0].qb200_last_error()


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(N=100), EINVAL, b"bad shape"),
    (dict(ld_u=68), EINVAL, b"row pitch"),
    (dict(ld_out=4097), EINVAL, b"row pitch"),
])
def test_expand_argument_errors(env, kw, rc, msg):
    assert _expand(env, **kw) == rc
    assert msg in env[0].qb200_last_error()


def test_problem_count_and_per_problem_pointers(env):
    p = env[3]
    for call in (_shrink, _expand):
        assert call(env, nprob=0) == EINVAL
        assert call(env, nprob=4) == EINVAL
        assert call(env, nprob=3, tables=(ct.c_void_p * 3)(p, p, None)) == EINVAL
        assert b"null pointer" in env[0].qb200_last_error()
        assert call(env, tables=(ct.c_void_p * 3)(p + 4, None, None)) == EINVAL
        assert b"aligned" in env[0].qb200_last_error()


def test_custom_op_is_registered():
    import torch

    import qlora_b200  # noqa: F401

    op = torch.ops.qlora_b200.lora_segmented_add.default
    assert [a.name for a in op._schema.arguments] == ["x2d", "tables", "rows", "n_adapters", "r", "outs"]
    assert op._schema.arguments[5].alias_info is not None and op._schema.arguments[5].alias_info.is_write


def test_names_form_branch_is_chosen_on_the_host():
    from qlora_b200.mixed import BASE_NAME, LoraAdapterSet, prefill_branch

    s = LoraAdapterSet.__new__(LoraAdapterSet)
    s.names = [f"a{i}" for i in range(5)]
    s.index = {n: i for i, n in enumerate(s.names)}
    s.ranks = [64, 64, 128, 8, 256]
    assert prefill_branch([s], ["a0", BASE_NAME, "a1", "a2"]) == "concat"            # 256
    assert prefill_branch([s], [BASE_NAME] * 3) == "concat"
    assert prefill_branch([s], ["a0", "a1", "a2", "a3"]) == "grouped"                # 264
    assert prefill_branch([s], ["a4", "a3"]) == "grouped"
