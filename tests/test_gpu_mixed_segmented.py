"""Mixed-adapter batches above 16 rows on the segmented path (qlora_b200/csrc/lora_segmented.cu): the base launch, U, a
segment table built on the device and the in-place tensor-core expand, with no read-back to the host.

* Against a float64 restatement on the C oracle's weights, with the bar of tests/test_gpu_mixed_adapters.py (for bf16 with a
  Frobenius bound that allows the path's second rounding, see `_check`): the row-index
  tensor form at 17, 64, 300 and 1600 rows (fused kernel, split-K, scratch path; U from the mixed projection and from the
  segmented shrink), 1, 3, 16 and 64 adapters of ranks 8, 16, 64 and 256 with interleaved base rows, 1000 adapters at the
  ragged shape, bf16 and fp16 compute, the 7B shapes, grouped q/k/v and gate/up.
* Bit for bit: base rows and out-of-range rows against the plain `Linear4bit` forward; permuting rows with their indices
  permutes the output.
* No host sync: an eager call under `torch.cuda.set_sync_debug_mode("error")`, and q/k/v + o captured in a CUDA graph at 64
  and 512 rows, replayed after the index buffer is rewritten.
* Reads stay inside each operand: NaN-padded adapters, index buffers whose neighbours point far outside the table.
* torch.compile(fullgraph=True) with a dynamic token count (tests/mixed_segmented_compile_case.py).
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from gpu_helpers import max_err_ulps, rel_err
from test_gpu_mixed_adapters import BF16, H16, SHAPES, _act, _adapters, _base, _names, _ref, _w64
from test_gpu_mixed_adapters import _check as _check_once

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOKENS = (17, 64, 300, 1600)
SEG_TOL_BF16 = 2.5e-3


def _check(y, ref, cdt):
    """fp16: the bar of the one-rounding paths.  bf16: each element within 1.01 ulp of max|ref| of the rounded reference, as
    there, and a Frobenius-relative bound of 2.5e-3 rather than 1e-3: the base output is rounded before the LoRA term is
    added, and the second rounding moves a share of the elements by one ulp.  Over the shapes, adapter counts and token
    counts of `test_tensor_form_matches_float64` the largest error measured on an H100 was 2.35e-3."""
    if cdt != BF16:
        return _check_once(y, ref, cdt)
    got, want = y.float().cpu().numpy(), ref.float().to(BF16).float().cpu().numpy()
    e, u = rel_err(got, want), max_err_ulps(got, want)
    assert e <= SEG_TOL_BF16 and u <= 1.01, f"rel_F={e:.3e}, max err = {u:.2f} bf16 ulp of max|ref|"


def _bnb():
    import qlora_b200 as q

    return q


def _rows(aset, names):
    return aset.indices(names)


# ---- 1. against float64 ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,k", SHAPES, ids=[f"{n}x{k}" for n, k in SHAPES])
def test_tensor_form_matches_float64(c_oracle, n, k, cdt):
    q = _bnb()
    base = _base(n, k, cdt, seed=n + k + 1)
    w64 = _w64(base, c_oracle, cdt)
    for na in (1, 3, 16, 64):
        adapters = _adapters(n, k, na, cdt, seed=100 * na + 7)
        aset = q.LoraAdapterSet(adapters)
        for m in TOKENS:
            names = _names(m, na)
            x = _act(m, k, seed=m + na, cdt=cdt)
            with torch.no_grad():
                y = q.lora_linear4bit_mixed(x, base, aset, _rows(aset, names))
            assert y.shape == (m, n) and y.dtype == cdt
            _check(y, _ref(x, w64, adapters, names, cdt), cdt)


@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
def test_thousand_adapters_matches_float64(c_oracle, cdt):
    """1000 adapters at the ragged shape: most tiles hold one or two rows, and every row may use a different adapter."""
    q = _bnb()
    n, k = 1000, 1088
    base = _base(n, k, cdt, seed=3)
    w64 = _w64(base, c_oracle, cdt)
    adapters = _adapters(n, k, 1000, cdt, seed=20000)
    aset = q.LoraAdapterSet(adapters)
    for m in TOKENS:
        names = _names(m, 1000)
        x = _act(m, k, seed=m, cdt=cdt)
        with torch.no_grad():
            y = q.lora_linear4bit_mixed(x, base, aset, _rows(aset, names))
        _check(y, _ref(x, w64, adapters, names, cdt), cdt)


@pytest.mark.parametrize("na", [6015, 6016, 7000])
def test_segment_table_histogram_in_shared_and_global_memory(c_oracle, na):
    """Rank-8 adapters at the ragged shape: 6015 adapters is the largest table whose counts the segment-table kernel keeps in
    shared memory; 6016 and 7000 take its global-memory histogram."""
    q = _bnb()
    n, k = 1000, 1088
    base = _base(n, k, BF16, seed=4)
    w64 = _w64(base, c_oracle, BF16)
    g = torch.Generator().manual_seed(na)
    a_all = ((torch.rand(na * 8, k, generator=g) * 2 - 1) * k ** -0.5).to(BF16).cuda()
    b_all = ((torch.rand(na, n, 8, generator=g) * 2 - 1) * 0.05).to(BF16).cuda()
    adapters = {f"ad{i}": (a_all[8 * i:8 * i + 8], b_all[i], 0.5 + 0.25 * (i % 3)) for i in range(na)}
    aset = q.LoraAdapterSet(adapters)
    for m in (300, 1600):
        names = ["__base__" if t % 3 == 1 else f"ad{(7919 * t) % na}" for t in range(m)]
        names[-1] = f"ad{na - 1}"
        x = _act(m, k, seed=m, cdt=BF16)
        with torch.no_grad():
            y = q.lora_linear4bit_mixed(x, base, aset, _rows(aset, names))
        _check(y, _ref(x, w64, adapters, names, BF16), BF16)


@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("group", ["qkv", "gate_up"])
def test_grouped_matches_float64(c_oracle, group, cdt):
    """q/k/v and gate/up, each linear with its own 16 adapters, one shared index tensor: one expand launch for all."""
    q = _bnb()
    n, k, p = (4096, 4096, 3) if group == "qkv" else (11008, 4096, 2)
    bases = [_base(n, k, cdt, seed=7 * i + 2) for i in range(p)]
    w64s = [_w64(b, c_oracle, cdt) for b in bases]
    adapters = [_adapters(n, k, 16, cdt, seed=1000 * (i + 1) + 5) for i in range(p)]
    sets = [q.LoraAdapterSet(a) for a in adapters]
    for m in (64, 1600):
        names = _names(m, 16)
        x = _act(m, k, seed=m, cdt=cdt)
        with torch.no_grad():
            ys = q.lora_linear4bit_group_mixed(x, bases, sets, _rows(sets[0], names))
        assert len(ys) == p
        for y, w64, ad in zip(ys, w64s, adapters):
            _check(y, _ref(x, w64, ad, names, cdt), cdt)


# ---- 2. bit for bit ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
def test_base_and_out_of_range_rows_are_linear4bit(cdt):
    q = _bnb()
    n, k = 4096, 4096
    base = _base(n, k, cdt, seed=5)
    aset = q.LoraAdapterSet(_adapters(n, k, 16, cdt, seed=50))
    for m in TOKENS:
        x = _act(m, k, seed=m, cdt=cdt)
        idx = [(t % 19) - 2 for t in range(m)]                   # -2, -1, 0..15, 16: three of every 19 rows have none
        idx[1::7] = [1 << 30] * len(idx[1::7])
        rows = torch.tensor(idx, dtype=torch.int32, device="cuda")
        with torch.no_grad():
            got = q.lora_linear4bit_mixed(x, base, aset, rows)
            plain = base(x)
            assert torch.equal(q.lora_linear4bit_mixed(x, base, aset, torch.full_like(rows, -1)), plain), m
        none = torch.tensor([t for t, a in enumerate(idx) if not 0 <= a < 16], device="cuda")
        assert torch.equal(got[none], plain[none]), m
        some = torch.tensor([t for t, a in enumerate(idx) if 0 <= a < 16], device="cuda")
        assert not torch.equal(got[some], plain[some]), m


def test_permuting_rows_permutes_the_output():
    q = _bnb()
    n, k = 4096, 4096
    base = _base(n, k, BF16, seed=8)
    aset = q.LoraAdapterSet(_adapters(n, k, 64, BF16, seed=80))
    for m in TOKENS:
        names = _names(m, 64)
        x = _act(m, k, seed=m, cdt=BF16)
        perm = torch.randperm(m, generator=torch.Generator().manual_seed(m)).cuda()
        rows = _rows(aset, names)
        with torch.no_grad():
            y = q.lora_linear4bit_mixed(x, base, aset, rows)
            yp = q.lora_linear4bit_mixed(x[perm].contiguous(), base, aset, rows[perm].contiguous())
        assert torch.equal(yp, y[perm]), m


# ---- 3. no host sync ---------------------------------------------------------------------------------------------------

def test_eager_call_does_not_sync():
    q = _bnb()
    n, k, m = 4096, 4096, 300
    bases = [_base(n, k, BF16, seed=60 + i) for i in range(3)]
    sets = [q.LoraAdapterSet(_adapters(n, k, 16, BF16, seed=600 + 50 * i)) for i in range(3)]
    x = _act(m, k, seed=1, cdt=BF16)
    rows = _rows(sets[0], _names(m, 16))
    with torch.no_grad():
        q.lora_linear4bit_group_mixed(x, bases, sets, rows)    # first call: library load, allocator growth
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ys = q.lora_linear4bit_group_mixed(x, bases, sets, rows)
            y = q.lora_linear4bit_mixed(ys[0], bases[0], sets[0], rows)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert bool(torch.isfinite(y).all())


@pytest.mark.parametrize("m", [64, 512])
def test_cuda_graph_replay_follows_the_index_buffer(m):
    """q/k/v (grouped) + o captured once; replays after writing all-base, one-adapter and 64-adapter assignments into the
    index buffer equal eager calls with those assignments."""
    q = _bnb()
    n, k = 4096, 4096
    bases = [_base(n, k, BF16, seed=11 + i) for i in range(4)]
    sets = [q.LoraAdapterSet(_adapters(n, k, 64, BF16, seed=300 + 40 * i)) for i in range(4)]
    x = _act(m, k, seed=1, cdt=BF16)
    rows = torch.zeros(m, dtype=torch.int32, device="cuda")
    assigns = [["__base__"] * m, ["ad5"] * m, [f"ad{(5 * t) % 64}" for t in range(m)]]

    def step(idx):
        ys = q.lora_linear4bit_group_mixed(x, bases[:3], sets[:3], idx)
        return list(ys) + [q.lora_linear4bit_mixed(ys[0], bases[3], sets[3], idx)]

    with torch.no_grad():
        sets[0].indices(assigns[2], out=rows)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(rows)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            outs = step(rows)
        results = []
        for assign in assigns:
            sets[0].indices(assign, out=rows)
            g.replay()
            want = step(sets[0].indices(assign))
            for a, b in zip(outs, want):
                assert torch.equal(a, b), assign[:3]
            results.append(outs[3].clone())
        assert not torch.equal(results[0], results[1]) and not torch.equal(results[1], results[2])


# ---- 4. reads stay inside each operand ---------------------------------------------------------------------------------

def test_reads_stay_inside_operands():
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
    for m in (17, 300):
        x = _act(m, k, seed=m, cdt=BF16)
        idx = [(t % 5) - 1 for t in range(m)]           # -1, 0, 1, 2, 3, -1, ...
        idx[0] = 1 << 30
        idx[-1] = -(1 << 31)
        buf = torch.full((m + 64,), -(1 << 30), dtype=torch.int32, device="cuda")
        buf[m + 32:] = (1 << 31) - 1
        buf[32:32 + m] = torch.tensor(idx, dtype=torch.int32)
        rows = buf[32:32 + m]
        with torch.no_grad():
            got = q.lora_linear4bit_mixed(x, base, pset, rows)
            want = q.lora_linear4bit_mixed(x, base, aset, rows)
            plain = base(x)
        assert bool(torch.isfinite(got).all()) and torch.equal(got, want), m
        for t, a in enumerate(idx):
            if not 0 <= a < 3:
                assert torch.equal(got[t], plain[t]), (m, t)


# ---- 5. torch.compile --------------------------------------------------------------------------------------------------

def test_compiled_segmented_has_one_graph_for_every_token_count():
    env = dict(os.environ)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mixed_segmented_compile_case.py")], capture_output=True,
                       text=True, env=env, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["graph_breaks"] == 0 and res["frames"] == 1, res
    assert all(res["equal"]) and res["assignments_differ"], res
