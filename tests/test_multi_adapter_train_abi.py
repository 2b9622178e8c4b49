"""The segmented backward's entry points without a GPU: they are declared and exported, their argument errors come back
before any launch, the custom ops are registered, and the shim exports the training entry points."""
import ctypes as ct
import os
import re

import pytest

EUNSUPPORTED, EINVAL = -2, -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("qb200_lora_grad_shrink_segmented", "qb200_lora_grad_input_segmented", "qb200_lora_weight_grad_segmented")


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
    integration = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    for name in NAMES:
        assert re.search(r"\bint " + name + r"\(", header), name
        assert name in L.EXPORTED_SYMBOLS and getattr(lib, name) is not None
        assert f"`{name}`" in integration, name


def _arrays(p, nprob):
    return (ct.c_void_p * max(3, nprob))(*([p] * nprob + [None] * (3 - nprob)))


def _grad_shrink(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, dY=_arrays(p, nprob), ld_dy=0, tables=_arrays(p, nprob), G=_arrays(p, nprob), ld_g=0, n=16, ws=p,
             ws_bytes=1 << 20, M=300, N=4096, R=64)
    a.update(kw)
    return lib.qb200_lora_grad_shrink_segmented(a["dtype"], nprob, a["dY"], a["ld_dy"], a["tables"], a["G"], a["ld_g"], a["n"],
                                                a["ws"], a["ws_bytes"], a["M"], a["N"], a["R"], None)


def _grad_input(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, accumulate=1, tables=_arrays(p, nprob), G=_arrays(p, nprob), ld_g=0, dx=_arrays(p, nprob), ld_dx=0, n=16,
             ws=p, ws_bytes=1 << 20, M=300, K=4096, R=64)
    a.update(kw)
    return lib.qb200_lora_grad_input_segmented(a["dtype"], nprob, a["accumulate"], a["tables"], a["G"], a["ld_g"], a["dx"],
                                               a["ld_dx"], a["n"], a["ws"], a["ws_bytes"], a["M"], a["K"], a["R"], None)


def _weight_grad(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, trans=0, tables=_arrays(p, nprob), offsets=p, total=64, P=_arrays(p, nprob), ld_p=0, Q=_arrays(p, nprob),
             ld_q=0, out=_arrays(p, nprob), n=16, ws=p, ws_bytes=1 << 20, M=300, D=4096, R=64)
    a.update(kw)
    return lib.qb200_lora_weight_grad_segmented(a["dtype"], nprob, a["trans"], a["tables"], a["offsets"], a["total"], a["P"],
                                                a["ld_p"], a["Q"], a["ld_q"], a["out"], a["n"], a["ws"], a["ws_bytes"], a["M"],
                                                a["D"], a["R"], None)


COMMON = [
    (dict(dtype=0), EINVAL, b"dtype"),
    (dict(tables=None), EINVAL, b"no null pointer"),
    (dict(ws=None), EINVAL, b"no null pointer"),
    (dict(n=0), EINVAL, b"n_adapters"),
    (dict(R=4), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(R=264), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(M=0), EINVAL, b"bad shape"),
    (dict(ws_bytes=256), EINVAL, b"workspace"),
    (dict(ws="p+8"), EINVAL, b"workspace"),
]


def _resolve(env, kw):
    p = env[3]
    return {k: (p + int(v[2:]) if isinstance(v, str) else v) for k, v in kw.items()}


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(G=None), EINVAL, b"no null pointer"),
    (dict(N=100), EINVAL, b"bad shape"),
    (dict(N=0), EINVAL, b"bad shape"),
    (dict(ld_dy=4100), EINVAL, b"row pitch"),
    (dict(ld_dy=4092), EINVAL, b"row pitch"),
    (dict(ld_g=32), EINVAL, b"row pitch"),
    (dict(ld_g=65), EINVAL, b"row pitch"),
])
def test_grad_shrink_argument_errors(env, kw, rc, msg):
    assert _grad_shrink(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(accumulate=2), EINVAL, b"accumulate"),
    (dict(dx=None), EINVAL, b"null pointer"),
    (dict(K=100), EINVAL, b"bad shape"),
    (dict(K=(65536 * 128)), EINVAL, b"bad shape"),
    (dict(ld_g=68), EINVAL, b"row pitch"),
    (dict(ld_g=32), EINVAL, b"row pitch"),
    (dict(ld_dx=4097), EINVAL, b"row pitch"),
    (dict(ld_dx=4000), EINVAL, b"row pitch"),
])
def test_grad_input_argument_errors(env, kw, rc, msg):
    assert _grad_input(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(trans=2), EINVAL, b"transpose_out"),
    (dict(offsets=None), EINVAL, b"null pointer"),
    (dict(offsets="p+4"), EINVAL, b"8-byte aligned"),
    (dict(Q=None), EINVAL, b"null pointer"),
    (dict(D=100), EINVAL, b"bad shape"),
    (dict(D=(65536 * 128)), EINVAL, b"bad shape"),
    (dict(total=0), EINVAL, b"rank_total"),
    (dict(ld_p=32), EINVAL, b"row pitch"),
    (dict(ld_q=4000), EINVAL, b"row pitch"),
])
def test_weight_grad_argument_errors(env, kw, rc, msg):
    assert _weight_grad(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


def test_problem_count_and_per_problem_pointers(env):
    p = env[3]
    for call in (_grad_shrink, _grad_input, _weight_grad):
        assert call(env, nprob=0) == EINVAL
        assert call(env, nprob=4) == EINVAL
        assert call(env, nprob=3, tables=(ct.c_void_p * 3)(p, p, None)) == EINVAL
        assert b"null pointer" in env[0].qb200_last_error()
        assert call(env, tables=(ct.c_void_p * 3)(p + 4, None, None)) == EINVAL
        assert b"aligned" in env[0].qb200_last_error()
    # the inputs each problem reads are checked per problem
    assert _grad_shrink(env, nprob=2, dY=(ct.c_void_p * 3)(p, p + 8, None)) == EINVAL
    assert b"aligned" in env[0].qb200_last_error()
    assert _weight_grad(env, nprob=2, Q=(ct.c_void_p * 3)(p, p + 8, None)) == EINVAL
    assert b"aligned" in env[0].qb200_last_error()
    assert _weight_grad(env, nprob=2, Q=(ct.c_void_p * 3)(p, None, None)) == EINVAL
    assert b"null pointer" in env[0].qb200_last_error()
    # accumulate = 1 reads dx[0] only; accumulate = 0 one output per problem
    assert _grad_input(env, nprob=3, dx=(ct.c_void_p * 3)(p, None, None), accumulate=0) == EINVAL
    assert b"null pointer" in env[0].qb200_last_error()


def test_workspace_size_restated_in_python(env):
    from qlora_b200 import _ops

    lib = env[0]
    for m, n in ((1, 1), (17, 1), (300, 16), (1600, 1000), (4097, 7000)):
        assert _ops.segment_workspace_bytes(m, n) == lib.qb200_lora_segment_workspace_size(m, n), (m, n)


def test_custom_ops_are_registered():
    import torch

    import qlora_b200  # noqa: F401

    fwd = torch.ops.qlora_b200.lora_segmented_fwd.default
    assert [a.name for a in fwd._schema.arguments] == ["xs", "tables", "rows", "n_adapters", "r", "outs"]
    assert fwd._schema.arguments[5].alias_info is not None and fwd._schema.arguments[5].alias_info.is_write
    assert len(fwd._schema.returns) == 2
    bwd = torch.ops.qlora_b200.lora_segmented_bwd.default
    assert [a.name for a in bwd._schema.arguments] == ["g2ds", "tables", "rank_offsets", "rank_total", "us", "xls", "ws",
                                                         "n_adapters", "r", "dx", "split"]
    assert bwd._schema.arguments[9].alias_info is not None and bwd._schema.arguments[9].alias_info.is_write
    assert len(bwd._schema.returns) == 3


def test_shim_exports_the_training_entry_points():
    import sys

    sys.path.insert(0, os.path.join(ROOT, "shims"))
    try:
        import bitsandbytes as bnb
    finally:
        sys.path.remove(os.path.join(ROOT, "shims"))
    import qlora_b200

    assert bnb.lora_linear4bit_group_multi is qlora_b200.lora_linear4bit_group_multi
    assert bnb.lora_linear4bit_multi is qlora_b200.lora_linear4bit_multi


def test_argument_errors_of_the_python_entry_points():
    """Raised on the host before any launch: host tensors (no CPU fallback), mismatched sets."""
    import torch

    from qlora_b200.mixed import lora_linear4bit_group_multi

    with pytest.raises(ValueError):
        lora_linear4bit_group_multi(torch.zeros(4, 8), [], [], torch.zeros(4, dtype=torch.int32))
