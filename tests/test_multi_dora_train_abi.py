"""Multi-adapter DoRA's entry points without a GPU: they are declared, exported and documented, their argument errors come
back before any launch, the custom ops are registered with the schemas the autograd function calls, the shim exports the
training entry points, and `DoraAdapterSet` is validated and refused by the LoRA entry points."""
import ctypes as ct
import os
import re

import pytest

EUNSUPPORTED, EINVAL = -2, -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("qb200_dora_stack_a", "qb200_dora_norm_segmented", "qb200_dora_expand_segmented", "qb200_dora_grad_scale_segmented")


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


def _stack(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, tables=_arrays(p, nprob), stack_rows=p, offsets=p, total=64, out=_arrays(p, nprob), n=4, K=4096, R=64)
    a.update(kw)
    return lib.qb200_dora_stack_a(a["dtype"], nprob, a["tables"], a["stack_rows"], a["offsets"], a["total"], a["out"], a["n"],
                                  a["K"], a["R"], None)


def _norm(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, tables=_arrays(p, nprob), mags=_arrays(p, nprob), offsets=p, gram_offsets=p, total=64, gram_total=4096,
             P=_arrays(p, nprob), norm2=_arrays(p, nprob), gram=_arrays(p, nprob), c=_arrays(p, nprob), nrm=_arrays(p, nprob),
             n=4, N=4096, K=4096, R=64)
    a.update(kw)
    return lib.qb200_dora_norm_segmented(a["dtype"], nprob, a["tables"], a["mags"], a["offsets"], a["gram_offsets"], a["total"],
                                         a["gram_total"], a["P"], a["norm2"], a["gram"], a["c"], a["nrm"], a["n"], a["N"], a["K"],
                                         a["R"], None)


def _expand(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, dropout=0, tables=_arrays(p, nprob), U=_arrays(p, nprob), ld_u=0, c=_arrays(p, nprob), Q=_arrays(p, nprob),
             out=_arrays(p, nprob), ld_out=0, n=16, ws=p, ws_bytes=1 << 20, M=300, N=4096, R=64)
    a.update(kw)
    return lib.qb200_dora_expand_segmented(a["dtype"], nprob, a["dropout"], a["tables"], a["U"], a["ld_u"], a["c"], a["Q"],
                                           a["out"], a["ld_out"], a["n"], a["ws"], a["ws_bytes"], a["M"], a["N"], a["R"], None)


def _scale(env, nprob=1, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, dropout=0, tables=_arrays(p, nprob), offsets=p, total=64, dY=_arrays(p, nprob), Q=_arrays(p, nprob),
             c=_arrays(p, nprob), nrm=_arrays(p, nprob), ld=0, dQ=_arrays(p, nprob), dD=_arrays(p, nprob), dm=_arrays(p, nprob),
             n=16, ws=p, ws_bytes=1 << 20, M=300, N=4096, R=64)
    a.update(kw)
    return lib.qb200_dora_grad_scale_segmented(a["dtype"], nprob, a["dropout"], a["tables"], a["offsets"], a["total"], a["dY"],
                                               a["Q"], a["c"], a["nrm"], a["ld"], a["dQ"], a["dD"], a["dm"], a["n"], a["ws"],
                                               a["ws_bytes"], a["M"], a["N"], a["R"], None)


CALLS = (_stack, _norm, _expand, _scale)
COMMON = [
    (dict(dtype=0), EINVAL, b"dtype"),
    (dict(dtype=3), EINVAL, b"dtype"),
    (dict(tables=None), EINVAL, b"no null pointer"),
    (dict(n=0), EINVAL, b"n_adapters"),
    (dict(R=4), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(R=12), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(R=264), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
]
SEGMENTED = [
    (dict(ws=None), EINVAL, b"no null pointer"),
    (dict(M=0), EINVAL, b"bad shape"),
    (dict(ws_bytes=256), EINVAL, b"workspace"),
    (dict(ws="p+8"), EINVAL, b"workspace"),
]


def _resolve(env, kw):
    p = env[3]
    return {k: (p + int(v[2:]) if isinstance(v, str) else v) for k, v in kw.items()}


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(stack_rows=None), EINVAL, b"null pointer"),
    (dict(offsets=None), EINVAL, b"null pointer"),
    (dict(out=None), EINVAL, b"null pointer"),
    (dict(out=(ct.c_void_p * 3)(8, None, None)), EINVAL, b"16-byte aligned"),
    (dict(offsets="p+4"), EINVAL, b"8-byte"),
    (dict(K=100), EINVAL, b"bad shape"),
    (dict(total=0), EINVAL, b"bad shape"),
])
def test_stack_argument_errors(env, kw, rc, msg):
    assert _stack(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


@pytest.mark.parametrize("kw,rc,msg", COMMON + [
    (dict(mags=None), EINVAL, b"null pointer"),
    (dict(P=None), EINVAL, b"null pointer"),
    (dict(gram=None), EINVAL, b"null pointer"),
    (dict(offsets=None), EINVAL, b"null pointer"),
    (dict(gram_offsets="p+4"), EINVAL, b"8-byte aligned"),
    (dict(c=(ct.c_void_p * 3)(4, None, None)), EINVAL, b"aligned"),
    (dict(N=100), EINVAL, b"bad shape"),
    (dict(N=0), EINVAL, b"bad shape"),
    (dict(gram_total=0), EINVAL, b"bad shape"),
])
def test_norm_argument_errors(env, kw, rc, msg):
    assert _norm(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


@pytest.mark.parametrize("kw,rc,msg", COMMON + SEGMENTED + [
    (dict(dropout=2), EINVAL, b"dropout"),
    (dict(U=None), EINVAL, b"no null pointer"),
    (dict(c=None), EINVAL, b"null pointer"),
    (dict(dropout=1, Q=None), EINVAL, b"null pointer"),
    (dict(N=100), EINVAL, b"bad shape"),
    (dict(ld_u=32), EINVAL, b"row pitch"),
    (dict(ld_out=4097), EINVAL, b"row pitch"),
])
def test_expand_argument_errors(env, kw, rc, msg):
    assert _expand(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


@pytest.mark.parametrize("kw,rc,msg", COMMON + SEGMENTED + [
    (dict(dropout=2), EINVAL, b"dropout"),
    (dict(dY=None), EINVAL, b"no null pointer"),
    (dict(dQ=None), EINVAL, b"no null pointer"),
    (dict(Q=None), EINVAL, b"null pointer"),
    (dict(dm=None), EINVAL, b"null pointer"),
    (dict(dropout=1, dD=None), EINVAL, b"null pointer"),
    (dict(offsets="p+4"), EINVAL, b"misaligned"),
    (dict(N=100), EINVAL, b"bad shape"),
    (dict(total=0), EINVAL, b"bad shape"),
    (dict(ld=4097), EINVAL, b"row pitch"),
    (dict(ld=4000), EINVAL, b"row pitch"),
])
def test_grad_scale_argument_errors(env, kw, rc, msg):
    assert _scale(env, **_resolve(env, kw)) == rc
    assert msg in env[0].qb200_last_error()


def test_problem_count_and_per_problem_pointers(env):
    p = env[3]
    for call in CALLS:
        assert call(env, nprob=0) == EINVAL
        assert call(env, nprob=4) == EINVAL
        assert b"1..3 problems" in env[0].qb200_last_error()
        assert call(env, nprob=3, tables=(ct.c_void_p * 3)(p, p, None)) == EINVAL
        assert b"null pointer" in env[0].qb200_last_error()
        assert call(env, tables=(ct.c_void_p * 3)(p + 4, None, None)) == EINVAL
        assert b"aligned" in env[0].qb200_last_error()
    # without dropout the expand and the gradient scale read no Q / dD
    assert _expand(env, nprob=2, c=(ct.c_void_p * 3)(p, None, None)) == EINVAL
    assert _scale(env, nprob=2, Q=(ct.c_void_p * 3)(p, None, None)) == EINVAL


def test_custom_ops_are_registered():
    import torch

    import qlora_b200  # noqa: F401

    ops = torch.ops.qlora_b200
    norm = ops.dora_segmented_norm.default._schema
    assert [a.name for a in norm.arguments] == ["tables", "mag_tables", "stack_rows", "rank_offsets", "gram_offsets", "rank_total",
                                                "gram_total", "packeds", "absmax", "code2", "absmax2", "offset", "n_out", "k_in",
                                                "state_dtype", "row_norm2s", "cdt", "n_adapters", "r"]
    assert len(norm.returns) == 2 and not any(a.alias_info is not None and a.alias_info.is_write for a in norm.arguments)
    fwd = ops.dora_segmented_fwd.default._schema
    assert [a.name for a in fwd.arguments] == ["xs", "tables", "rows", "n_adapters", "r", "cs", "outs", "qs"]
    assert [a.name for a in fwd.arguments if a.alias_info is not None and a.alias_info.is_write] == ["outs", "qs"]
    assert len(fwd.returns) == 2
    scale = ops.dora_grad_scale.default._schema
    assert [a.name for a in scale.arguments] == ["g2ds", "tables", "rank_offsets", "rank_total", "qs", "cs", "nrms", "ws",
                                                 "n_adapters", "r", "split"]
    assert len(scale.returns) == 3
    bwd = ops.dora_segmented_bwd.default._schema
    assert [a.name for a in bwd.arguments] == ["dqs", "tables", "rank_offsets", "rank_total", "us", "xls", "ws", "n_adapters", "r",
                                               "dxs"]
    assert [a.name for a in bwd.arguments if a.alias_info is not None and a.alias_info.is_write] == ["dxs"]
    assert len(bwd.returns) == 2


def test_shim_exports_the_training_entry_points():
    import sys

    sys.path.insert(0, os.path.join(ROOT, "shims"))
    try:
        import bitsandbytes as bnb
    finally:
        sys.path.remove(os.path.join(ROOT, "shims"))
    import qlora_b200

    assert bnb.DoraAdapterSet is qlora_b200.DoraAdapterSet
    assert bnb.dora_linear4bit_group_multi is qlora_b200.dora_linear4bit_group_multi
    assert bnb.dora_linear4bit_multi is qlora_b200.dora_linear4bit_multi


def test_dora_adapter_set_validation():
    import torch

    from qlora_b200.mixed import DoraAdapterSet, LoraAdapterSet

    assert issubclass(DoraAdapterSet, LoraAdapterSet)
    a, b, m = torch.zeros(8, 64, dtype=torch.bfloat16), torch.zeros(32, 8, dtype=torch.bfloat16), torch.ones(32, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="no adapters"):
        DoraAdapterSet({})
    with pytest.raises(ValueError, match="magnitude"):
        DoraAdapterSet({"x": (a, b, 1.0)})                    # a LoRA entry: no magnitude
    with pytest.raises(ValueError, match="__base__"):
        DoraAdapterSet({"__base__": (a, b, m, 1.0)})
    with pytest.raises(ValueError, match="CUDA"):
        DoraAdapterSet({"x": (a, b, m, 1.0)})                 # host tensors: no CPU fallback


def test_lora_entry_points_refuse_a_dora_set():
    """A DoraAdapterSet passed to the LoRA entry points raises instead of silently dropping its magnitudes."""
    import torch

    from qlora_b200 import mixed

    s = object.__new__(mixed.DoraAdapterSet)                  # no device needed: the refusal comes first
    x, rows = torch.zeros(4, 64), torch.zeros(4, dtype=torch.int32)
    for call in (lambda: mixed.lora_linear4bit_group_mixed(x, [None], [s], rows),
                 lambda: mixed.lora_linear4bit_mixed(x, None, s, rows),
                 lambda: mixed.lora_linear4bit_group_multi(x, [None], [s], rows),
                 lambda: mixed.lora_linear4bit_multi(x, None, s, rows)):
        with pytest.raises(ValueError, match="DoraAdapterSet"):
            call()
    # and the DoRA entry points take DoraAdapterSets only
    plain = object.__new__(mixed.LoraAdapterSet)
    with pytest.raises(ValueError, match="DoraAdapterSet"):
        mixed.dora_linear4bit_group_multi(x, [None], [plain], rows)
    with pytest.raises(ValueError, match="DoraAdapterSet"):
        mixed.dora_linear4bit_multi(x, None, plain, rows)
