"""Mixed-adapter batches without a GPU: the two entry points are declared and exported, their argument errors come back
before any launch, adapter names are validated on the host, and the path refuses to run in grad mode."""
import ctypes as ct
import os
import re
import types

import pytest
import torch

EUNSUPPORTED, EINVAL = -2, -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("qb200_lora_project_mixed", "qb200_nf4_linear_group_mixed")


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
    assert "typedef struct qb200_lora_adapter" in header
    assert ct.sizeof(L.LoraAdapter) == 24


def _project(env, **kw):
    lib, _, _, p = env
    a = dict(dtype=2, x=p, ld_x=0, table=p, n=4, rows=p, u=p, ld_u=0, M=4, K=128, R=64)
    a.update(kw)
    return lib.qb200_lora_project_mixed(a["dtype"], a["x"], a["ld_x"], a["table"], a["n"], a["rows"], a["u"], a["ld_u"], a["M"],
                                        a["K"], a["R"], None)


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(dtype=0), EINVAL, b"dtype"),
    (dict(x=None), EINVAL, b"null pointer"),
    (dict(table=None), EINVAL, b"null pointer"),
    (dict(rows=None), EINVAL, b"null pointer"),
    (dict(n=0), EINVAL, b"n_adapters"),
    (dict(M=0), EINVAL, b"bad shape"),
    (dict(K=100), EINVAL, b"bad shape"),
    (dict(R=4), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(R=264), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(ld_u=32), EINVAL, b"row pitch"),
    (dict(ld_x=100), EINVAL, b"row pitch"),
])
def test_project_mixed_argument_errors(env, kw, rc, msg):
    assert _project(env, **kw) == rc
    assert msg in env[0].qb200_last_error()


def test_project_mixed_alignment(env):
    p = env[3]
    assert _project(env, x=p + 2) == EINVAL
    assert _project(env, table=p + 4) == EINVAL
    assert b"aligned" in env[0].qb200_last_error()


def _group(env, nprob=1, with_table=True, **kw):
    lib, L, _, p = env
    pr = L.Nf4Problem(inp=p, packed=p, absmax_f32=p, out=p, U=p, V=p if with_table else None)
    probs = (L.Nf4Problem * 3)(pr, pr, pr)
    a = dict(dtype=2, state=2, n=4, rows=p, R=64, M=8, N=128, K=128, out=2)
    a.update(kw)
    return lib.qb200_nf4_linear_group_mixed(a["dtype"], a["state"], nprob, ct.addressof(probs), a["n"], a["rows"], a["R"], a["M"],
                                            a["N"], a["K"], a["out"], None)


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(dtype=0), EINVAL, b"unsupported (dtype"),
    (dict(dtype=1, state=2), EINVAL, b"unsupported (dtype"),
    (dict(out=0), EUNSUPPORTED, b"16-bit outputs"),
    (dict(rows=None), EINVAL, b"row_adapter"),
    (dict(n=0), EINVAL, b"no adapters"),
    (dict(M=17), EUNSUPPORTED, b"skinny token counts"),
    (dict(K=100), EUNSUPPORTED, b"multiple of 64"),
    (dict(R=0), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
    (dict(R=72 + 4), EUNSUPPORTED, b"multiple of 8 in [8, 256]"),
])
def test_group_mixed_argument_errors(env, kw, rc, msg):
    assert _group(env, **kw) == rc
    assert msg in env[0].qb200_last_error()


def test_group_mixed_needs_tables_and_problem_count(env):
    assert _group(env, with_table=False) == EINVAL
    assert b"null LoRA operand" in env[0].qb200_last_error()
    assert _group(env, nprob=0) == EINVAL
    assert _group(env, nprob=4) == EINVAL


def _fake_set(names):
    from qlora_b200.mixed import LoraAdapterSet

    s = LoraAdapterSet.__new__(LoraAdapterSet)
    s.names = list(names)
    s.index = {n: i for i, n in enumerate(names)}
    s.device = torch.device("cpu")
    s.lora_as, s.lora_bs = [], []
    return s


def test_names_are_validated_on_the_host():
    s = _fake_set(["math", "code", "chat"])
    assert s.indices(["code", "__base__", "chat", "math", "code"]).tolist() == [1, -1, 2, 0, 1]
    with pytest.raises(ValueError, match="non-existing adapter"):
        s.indices(["code", "poetry"])
    out = torch.zeros(3, dtype=torch.int32)
    s.indices(["chat", "chat", "__base__"], out=out)
    assert out.tolist() == [2, 2, -1]


def test_base_name_is_not_an_adapter():
    from qlora_b200.mixed import LoraAdapterSet

    with pytest.raises(ValueError, match="__base__"):
        LoraAdapterSet({"__base__": (None, None, 1.0)})
    with pytest.raises(ValueError, match="no adapters"):
        LoraAdapterSet({})


def test_grad_mode_is_refused():
    import qlora_b200 as q

    s = _fake_set(["a"])
    s.lora_as = [torch.zeros(8, 64, requires_grad=True)]
    x = torch.zeros(2, 64)
    base = types.SimpleNamespace()
    with pytest.raises(RuntimeError, match="inference only"):
        q.lora_linear4bit_mixed(x, base, s, ["a", "__base__"])
    with pytest.raises(RuntimeError, match="inference only"):
        q.lora_linear4bit_mixed(x.requires_grad_(), base, _fake_set(["a"]), ["a", "a"])


def test_shim_exports():
    import importlib
    import sys

    sys.path.insert(0, os.path.join(ROOT, "shims"))
    try:
        bnb = importlib.import_module("bitsandbytes")
    finally:
        sys.path.remove(os.path.join(ROOT, "shims"))
    for name in ("LoraAdapterSet", "lora_linear4bit_mixed", "lora_linear4bit_group_mixed"):
        assert hasattr(bnb, name), name
