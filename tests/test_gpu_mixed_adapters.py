"""Mixed-adapter batches over the NF4 base (qlora_b200/mixed.py): every token row with its own LoRA adapter, "__base__" rows
with none.

* Against a float64 restatement on the C oracle's weights (the bar of tests/test_gpu_lora_rank.py): 7B shapes and a ragged
  one, 1, 2, 5 and 16 tokens (decode: the mixed projection and skinny kernels) and 1600 (the scratch path under bf16
  compute), 1, 3, 16 and 64 adapters of ranks 8, 16, 64 and 256 with interleaved base rows, bf16 and fp16 compute, both
  prefill branches, grouped q/k/v and gate/up.
* Bit for bit: a batch that uses one adapter against `lora_linear4bit` with it (decode and concat prefill), base rows
  against the plain `Linear4bit` forward.
* A captured CUDA graph replayed after its row-index buffer is overwritten, against eager.
* Reads stay inside each operand: padded adapters in NaN buffers, row indices outside the table.
* torch.compile(fullgraph=True) of a 2-layer HF-built model's mixed decode forward (tests/mixed_compile_case.py): no graph
  break, and eager's bits under the aot_eager backend.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fp16_helpers import assert_close_f16, f16_round, oracle_w16
from gpu_helpers import assert_close_bf16, make_act, make_weight, oracle_weight

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, H16, F32 = torch.bfloat16, torch.float16, torch.float32
TOL = 1e-3
RANKS = [8, 16, 64, 256]
SHAPES = [(4096, 4096), (11008, 4096), (4096, 11008), (1000, 1088)]   # (N, K)


def _bnb():
    import qlora_b200 as q

    return q


def _base(n, k, cdt, seed):
    q = _bnb()
    lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=cdt, quant_type="nf4")
    lin.weight = q.nn.Params4bit(make_weight(n, k, seed=seed, dtype=cdt), requires_grad=False, compress_statistics=True,
                                 quant_type="nf4", module=lin)
    return lin.cuda()


def _adapters(n, k, na, cdt, seed):
    """{name: (A, B, scaling)}: adapter i has rank RANKS[i % 4]."""
    out = {}
    for i in range(na):
        r = RANKS[i % len(RANKS)]
        a = make_weight(r, k, seed=seed + 2 * i, dtype=cdt, scale=k ** -0.5)
        b = make_weight(n, r, seed=seed + 2 * i + 1, dtype=cdt, scale=0.05)
        out[f"ad{i}"] = (a, b, 0.5 + 0.25 * (i % 3))
    return out


def _names(m, na):
    return ["__base__" if t % 3 == 1 else f"ad{(7 * t) % na}" for t in range(m)]


def _w64(base, c_oracle, cdt):
    w = base.weight
    if cdt == BF16:
        return torch.from_numpy(oracle_weight(w.data, w.quant_state, c_oracle)).cuda().double()
    return torch.from_numpy(oracle_w16(c_oracle, w.data, w.quant_state)).cuda().double()


def _ref(x, w64, adapters, names, cdt):
    """float64: x W^T + U B^T per row, U = scaling x A^T rounded once to the compute dtype."""
    x64 = x.double()
    y = x64 @ w64.t()
    for name, (a, b, s) in adapters.items():
        sel = torch.tensor([t for t, nm in enumerate(names) if nm == name], dtype=torch.long, device=x.device)
        if sel.numel() == 0:
            continue
        u = (s * (x64[sel] @ a.double().t())).to(cdt).double()
        y[sel] += u @ b.double().t()
    return y


def _check(y, ref, cdt):
    got = y.float().cpu().numpy()
    if cdt == BF16:
        assert_close_bf16(got, ref.float().to(BF16).float().cpu().numpy(), TOL)
    else:
        assert_close_f16(got, f16_round(ref.float().cpu().numpy()), TOL)


def _act(m, k, seed, cdt):
    return make_act(m, k, seed=seed).to(cdt)


# ---- 1. against float64 ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,k", SHAPES, ids=[f"{n}x{k}" for n, k in SHAPES])
def test_matches_float64(c_oracle, n, k, cdt):
    """Every (adapter count, token count): the decode kernels at 1..16 tokens, and at 1600 tokens the concat branch (1 and 3
    adapters: ranks add up to 8 and 88) or the grouped fallback (16 and 64 adapters)."""
    q = _bnb()
    base = _base(n, k, cdt, seed=n + k)
    w64 = _w64(base, c_oracle, cdt)
    for na in (1, 3, 16, 64):
        adapters = _adapters(n, k, na, cdt, seed=100 * na)
        aset = q.LoraAdapterSet(adapters)
        for m in (1, 2, 5, 16, 1600):
            names = _names(m, na)
            if m == 1:
                names = [f"ad{na - 1}"]
            x = _act(m, k, seed=m + na, cdt=cdt)
            with torch.no_grad():
                y = q.lora_linear4bit_mixed(x, base, aset, names)
            assert y.shape == (m, n) and y.dtype == cdt
            _check(y, _ref(x, w64, adapters, names, cdt), cdt)
            if m == 1600:
                from qlora_b200.mixed import prefill_branch

                assert prefill_branch([aset], names) == ("concat" if na <= 3 else "grouped")


@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("group", ["qkv", "gate_up"])
def test_grouped_matches_float64(c_oracle, group, cdt):
    """q/k/v (3 x 4096x4096) and gate/up (2 x 11008x4096), each linear with its own 16 adapters of one set of names."""
    q = _bnb()
    n, k, p = (4096, 4096, 3) if group == "qkv" else (11008, 4096, 2)
    bases = [_base(n, k, cdt, seed=7 * i + 1) for i in range(p)]
    w64s = [_w64(b, c_oracle, cdt) for b in bases]
    adapters = [_adapters(n, k, 16, cdt, seed=1000 * (i + 1)) for i in range(p)]
    sets = [q.LoraAdapterSet(a) for a in adapters]
    for m in (5, 16, 1600):
        names = _names(m, 16)
        x = _act(m, k, seed=m, cdt=cdt)
        with torch.no_grad():
            ys = q.lora_linear4bit_group_mixed(x, bases, sets, names)
        assert len(ys) == p
        for y, w64, ad in zip(ys, w64s, adapters):
            _check(y, _ref(x, w64, ad, names, cdt), cdt)


# ---- 2. bit for bit ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
def test_one_adapter_is_lora_linear4bit_and_base_rows_are_linear4bit(cdt):
    """All rows on adapter "ad2" (rank 64, of a set of three) give `lora_linear4bit`'s bits at decode token counts and at
    300 and 1600 tokens (concat branch: fused kernel, scratch path); "__base__" rows, alone or interleaved with adapter
    rows, give the plain `Linear4bit` forward's bits."""
    q = _bnb()
    n, k = 4096, 4096
    base = _base(n, k, cdt, seed=5)
    adapters = _adapters(n, k, 3, cdt, seed=50)
    aset = q.LoraAdapterSet(adapters)
    a, b, s = adapters["ad2"]
    for m in (1, 5, 16, 300, 1600):
        x = _act(m, k, seed=m, cdt=cdt)
        with torch.no_grad():
            got = q.lora_linear4bit_mixed(x, base, aset, ["ad2"] * m)
            want = q.lora_linear4bit(x, base, a, b, s)
            assert torch.equal(got, want), m
            plain = base(x)
            assert torch.equal(q.lora_linear4bit_mixed(x, base, aset, ["__base__"] * m), plain), m
            names = _names(m, 3)
            mixed = q.lora_linear4bit_mixed(x, base, aset, names)
            sel = torch.tensor([t for t, nm in enumerate(names) if nm == "__base__"], dtype=torch.long, device="cuda")
            assert torch.equal(mixed[sel], plain[sel]), m


# ---- 3. CUDA graph -----------------------------------------------------------------------------------------------------

def test_cuda_graph_replay_follows_the_index_buffer():
    """A decode step of q/k/v + o (grouped and single) captured once; replays after copying new assignments into its
    row-index buffer equal eager calls with those assignments."""
    q = _bnb()
    n, k, m = 4096, 4096, 8
    bases = [_base(n, k, BF16, seed=11 + i) for i in range(4)]
    sets = [q.LoraAdapterSet(_adapters(n, k, 5, BF16, seed=300 + 40 * i)) for i in range(4)]
    x = _act(m, k, seed=1, cdt=BF16)
    rows = torch.zeros(m, dtype=torch.int32, device="cuda")
    assigns = [_names(m, 5), ["ad4"] * m, ["__base__", "ad0", "ad1", "ad2", "ad3", "ad4", "ad0", "__base__"]]

    def step(idx):
        ys = q.lora_linear4bit_group_mixed(x, bases[:3], sets[:3], idx)
        return list(ys) + [q.lora_linear4bit_mixed(ys[0], bases[3], sets[3], idx)]

    with torch.no_grad():
        sets[0].indices(assigns[0], out=rows)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(rows)                       # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            outs = step(rows)
        for assign in assigns[::-1]:
            sets[0].indices(assign, out=rows)
            g.replay()
            want = step(assign)
            for a, b in zip(outs, want):
                assert torch.equal(a, b), assign


# ---- 4. reads stay inside each operand ---------------------------------------------------------------------------------

def test_reads_stay_inside_operands():
    """Adapters as the leading rows of NaN-filled buffers, the row indices a slice of a buffer whose other entries index far
    outside the table, and indices outside [0, 3) inside the slice: every output is finite, equals the call on unpadded
    adapters, and a row with an out-of-range index equals a base row."""
    q = _bnb()
    n, k = 1000, 1088
    base = _base(n, k, BF16, seed=9)
    adapters = _adapters(n, k, 3, BF16, seed=70)

    def padded(t):
        buf = torch.full((t.shape[0] + 64, t.shape[1]), float("nan"), dtype=t.dtype, device="cuda")
        buf[:t.shape[0]] = t
        return buf[:t.shape[0]]

    pset = q.LoraAdapterSet({nm: (padded(a), padded(b), s) for nm, (a, b, s) in adapters.items()})
    aset = q.LoraAdapterSet(adapters)
    for m in (1, 5, 16):
        x = _act(m, k, seed=m, cdt=BF16)
        idx = [(t % 5) - 1 for t in range(m)]           # -1, 0, 1, 2, 3, -1, ...
        idx[0] = 1 << 30 if m > 1 else idx[0]
        buf = torch.full((m + 32,), -(1 << 30), dtype=torch.int32, device="cuda")
        buf[m:] = 1 << 30
        buf[:m] = torch.tensor(idx, dtype=torch.int32)
        rows = buf[:m]
        with torch.no_grad():
            got = q.lora_linear4bit_mixed(x, base, pset, rows)
            want = q.lora_linear4bit_mixed(x, base, aset, rows)
            plain = base(x)
        assert bool(torch.isfinite(got).all()) and torch.equal(got, want), m
        for t, a in enumerate(idx):
            if not 0 <= a < 3:
                assert torch.equal(got[t], plain[t]), (m, t)


# ---- 5. torch.compile --------------------------------------------------------------------------------------------------

def test_compiled_mixed_decode_has_no_graph_break():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "shims") + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mixed_compile_case.py")], capture_output=True, text=True,
                       env=env, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for backend in ("aot_eager", "inductor"):
        got = res[backend]
        assert got["graph_breaks"] == 0 and got["frames"] == 1 and got["assignments_differ"], res
    # the traced graph run op by op gives eager's bits; inductor's own kernels for the non-linear glue round differently
    assert all(res["aot_eager"]["equal"]), res
    assert max(res["inductor"]["rel_vs_eager"]) < 2e-2, res
