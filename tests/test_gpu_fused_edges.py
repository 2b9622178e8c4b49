"""The fused NF4 kernel (nf4_gemm_wgmma_kernel) below the scratch path's token counts, at the edges of its two schedules: the
range schedule, and split-K (fp32 partials of every tile's contraction in a lent workspace, then splitk_reduce_kernel).
Every call with 17 to 1535 tokens runs one of them, as do fp16 compute, fp16 states, fp16 outputs and row-scaled calls at
every token count.

Checked against the C oracle's weights in float64, rounded once: ragged feature and contraction tails (a last feature tile
8 wide, a last contraction block of 8 rows inside a shorter last split), LoRA ranks that end inside a 64-wide step, grouped
launches whose problems meet inside one CTA's range, operands padded with NaN where a correct kernel never reads, outputs
that are pitched or offset views of sentinel-filled buffers, non-power-of-two row scales (bit for bit, with identity
inputs), and calls chained without host syncs, eagerly and from a CUDA graph.  Every case asserts which schedule it took;
the token counts are classified by the library's own plan, which depends on the SM count."""
import ctypes as ct
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import fused_kernel_names_case as names_case
import fused_splitk_case as case
import oracle_c as oc
from gpu_helpers import assert_close_bf16, make_act, make_weight, oracle_weight, state_to_numpy
from oracle import nf4_oracle as o

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, H16, F32 = torch.bfloat16, torch.float16, torch.float32
TOL = 1e-3
# (N, K): 65 contraction blocks for dX (the last 8 rows) and a last forward feature tile 8 wide | 172 dX blocks (the last 56
# rows), 86 forward feature tiles | 16 dX blocks (the last 40 rows), a last forward feature tile 104 wide | 3 blocks each way
SHAPES = [(4104, 4160), (11000, 1088), (1000, 1088), (200, 192)]
SHAPE_IDS = ["x".join(map(str, s)) for s in SHAPES]
# token counts at unit edges: one past 16, 32, 128 and 256, inside a tile, and the last below the scratch path
TOKENS = [17, 33, 100, 129, 257, 777, 1000, 1535]
RANKS = [8, 24, 56, 72, 136]
SCRATCH_MIN_M = 1536


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    return F


def _lib():
    from qlora_b200 import _lib

    return _lib.load()


def _workspace(m, n, k, is_bwd):
    return _lib().qb200_nf4_linear_workspace_size(m, n, k, int(is_bwd))


def _schedule(m, n, k, is_bwd):
    """The kernel a single-problem call with a 16-bit output takes: 'skinny', 'splitk' or 'range'."""
    if not is_bwd and m <= 16:
        assert _workspace(m, n, k, is_bwd) == 0
        return "skinny"
    if _workspace(m, n, k, is_bwd) > 0:
        return "splitk"
    assert m < SCRATCH_MIN_M and _lib().qb200_nf4_linear_scratch_size(1, m, n, k, int(is_bwd)) == 0
    return "range"


def _ksplit(m, n, k, is_bwd):
    """Splits the library plans (the workspace holds ksplit fp32 [M, F] partials)."""
    return _workspace(m, n, k, is_bwd) // (m * (k if is_bwd else n) * 4)


def _tokens_for(schedule, n=4104, k=4160, directions=(False, True)):
    """The first of TOKENS that takes `schedule` in every direction given."""
    for m in TOKENS:
        if all(_schedule(m, n, k, d) == schedule for d in directions):
            return m
    pytest.fail(f"no token count of {TOKENS} takes the {schedule} schedule at {n}x{k}")


def _quant(F, n, k, seed, nested=True, state_dtype=BF16):
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=seed, dtype=state_dtype), compress_statistics=nested, quant_type="nf4")
    assert qs.dtype == state_dtype
    return packed.t(), qs


def _w64(packed, qs, c_oracle):
    """The oracle's bf16 weight [N, K] as float64 on the GPU."""
    return torch.from_numpy(oracle_weight(packed, qs, c_oracle)).cuda().double()


def _restated_weight(c_oracle, packed, qs, table, scale=None):
    """W [N, K] restated in numpy float32: the oracle's fp32 absmax of every block, times its row's scale (one correctly
    rounded fp32 multiply, as __fmul_rn), then LUT[j] * absmax rounded to `table` ('bf16' or 'fp16')."""
    st = state_to_numpy(packed, qs)
    n, k = st["shape"]
    if st["nested"]:
        am = oc.nested_absmax(c_oracle, st["code256"], st["absmax_u8"], st["absmax2"], st["offset"])
    else:
        am = st["absmax"].astype(np.float32)
    if scale is not None:
        am = (am.reshape(n, k // 64) * scale.cpu().numpy().astype(np.float32)[:, None]).astype(np.float32).reshape(-1)
    return o.dequantize_nf4(st["packed"], am, n * k, 64, table).reshape(n, k)


def _check(y, ref64, dtype=BF16):
    """The parity bar against a float64 reference rounded to `dtype` once (bf16 then fp16 for an fp16 output under bf16
    compute, as the kernel rounds it)."""
    ref = ref64.float().to(BF16) if dtype == BF16 else ref64.float().to(H16)
    if y.dtype != ref.dtype:
        ref = ref.to(y.dtype)
    assert_close_bf16(y.float().cpu().numpy(), ref.float().cpu().numpy(), TOL)


def _nan_buffer(rows, cols, dtype=BF16):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device="cuda")


def _padded(t, extra_rows=256, extra_cols=64):
    """`t` [R, C] as the top-left view of an [R + extra_rows, C + extra_cols] buffer that is NaN elsewhere."""
    buf = _nan_buffer(t.shape[0] + extra_rows, t.shape[1] + extra_cols, t.dtype)
    buf[:t.shape[0], :t.shape[1]] = t
    return buf[:t.shape[0], :t.shape[1]]


def _prefix(t, fill, extra=4096):
    """Contiguous `t` as the prefix of a flat allocation `extra` elements longer, filled with `fill` after it."""
    buf = torch.full((t.numel() + extra,), fill, dtype=t.dtype, device="cuda")
    buf[:t.numel()] = t.reshape(-1)
    return buf[:t.numel()].view(t.shape)


def _state_ptrs(F, qs):
    return tuple(None if t is None else t.data_ptr() for t in F._state_tensors(qs, torch.device("cuda")))


def _group_ex(F, is_bwd, x, packed, qs, out, ws, cdt=BF16, out_dtype=BF16, bias=None):
    """`qb200_nf4_linear_group_ex` for one problem writing the caller's `out`, with workspace `ws` (None: none)."""
    from qlora_b200._lib import DTYPE_CODE, Nf4Problem

    n, k = qs.shape
    pr = Nf4Problem(inp=x.data_ptr(), ld_in=x.stride(0), packed=packed.data_ptr(), bias=None if bias is None else bias.data_ptr(),
                    out=out.data_ptr(), ld_out=out.stride(0))
    pr.absmax_u8, pr.code256, pr.absmax2, pr.offset, pr.absmax_f32 = _state_ptrs(F, qs)
    probs = (Nf4Problem * 1)(pr)
    rc = _lib().qb200_nf4_linear_group_ex(int(is_bwd), DTYPE_CODE[cdt], DTYPE_CODE[qs.dtype], 1, ct.addressof(probs), 0, x.shape[0],
                                          n, k, DTYPE_CODE[out_dtype], None if ws is None else ws.data_ptr(),
                                          0 if ws is None else ws.numel(), F.stream_ptr(x.device))
    assert rc == 0, _lib().qb200_last_error()
    return out


# ---- 1. parity with the oracle at ragged shapes ------------------------------------------------------------------------

def test_token_counts_reach_both_schedules(F):
    """The parametrization below reaches split-K and the range schedule in both directions, and split-K at its edges: a dX
    over 65 contraction blocks that the splits do not divide (the last block 8 rows, inside the last split) and a forward
    whose last feature tile is 8 wide."""
    reached = {(is_bwd, _schedule(m, n, k, is_bwd)) for n, k in SHAPES for m in TOKENS for is_bwd in (False, True)}
    assert reached == {(False, "splitk"), (False, "range"), (True, "splitk"), (True, "range")}, reached
    ks_dx = [_ksplit(m, 4104, 4160, True) for m in TOKENS if _schedule(m, 4104, 4160, True) == "splitk"]
    assert any(65 % ks != 0 for ks in ks_dx), ks_dx
    assert any(_schedule(m, 4104, 4160, False) == "splitk" for m in TOKENS)


STATES = [(True, BF16), (False, BF16), (True, F32)]
STATE_IDS = ["nested", "plain", "f32state"]


@pytest.mark.parametrize("nested,state_dtype", STATES, ids=STATE_IDS)
@pytest.mark.parametrize("n,k", SHAPES, ids=SHAPE_IDS)
def test_fused_matches_oracle_at_ragged_shapes(F, c_oracle, n, k, nested, state_dtype):
    """At every token count of TOKENS: forward with bias, forward with LoRA and bias, dX with LoRA (the rank cycling through
    RANKS), each on the schedule the library plans; fp32 outputs are the bf16 outputs widened."""
    packed, qs = _quant(F, n, k, seed=n + k, nested=nested, state_dtype=state_dtype)
    w = _w64(packed, qs, c_oracle)
    x_all, dy_all = make_act(max(TOKENS), k, seed=1), make_act(max(TOKENS), n, seed=2)
    bias = make_weight(1, n, seed=3, scale=0.5).view(-1)
    for j, m in enumerate(TOKENS):
        assert _schedule(m, n, k, False) in ("splitk", "range") and _schedule(m, n, k, True) in ("splitk", "range")
        r = RANKS[(j + SHAPES.index((n, k))) % len(RANKS)]
        x, dy = x_all[:m], dy_all[:m]
        base = x.double() @ w.t() + bias.double()
        y = F.nf4_linear_fwd(x, packed, qs, bias)
        _check(y, base)
        assert torch.equal(F.nf4_linear_fwd(x, packed, qs, bias, out_dtype=F32), y.float()), m
        u, v = make_act(m, r, seed=10 + j), make_weight(n, r, seed=20 + j, scale=0.05)
        yl = F.nf4_linear_fwd_lora(x, packed, qs, u, v, bias)
        _check(yl, base + u.double() @ v.double().t())
        assert torch.equal(F.nf4_linear_fwd_lora(x, packed, qs, u, v, bias, out_dtype=F32), yl.float()), m
        g, a = make_act(m, r, seed=30 + j), make_weight(r, k, seed=40 + j, scale=0.05)
        dx = F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a)
        _check(dx, dy.double() @ w + g.double() @ a.double())
        assert torch.equal(F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a, out_dtype=F32), dx.float()), m


def test_split_k_with_uneven_splits_matches_oracle(F, c_oracle, tmp_path):
    """fused_splitk_case.py run with all but 32 SMs reserved: the planner then splits the contraction 2 to 4 ways with a
    shorter last split.  Each output of the subprocess is checked against the oracle."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert sms - 32 > 0
    env = dict(os.environ, QB200_RESERVED_SMS=str(sms - 32))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "fused_splitk_case.py"), str(tmp_path / "out.npz")],
                       capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    uneven = 0
    for n, k, m, rank in case.CASES:
        key = f"{n}x{k}_{m}"
        for is_bwd, f_out, c in ((False, n, k), (True, k, n)):
            ks = int(got[key + ("_dx_ws" if is_bwd else "_fwd_ws")]) // (m * f_out * 4)
            num_kb = -(-c // 64)
            per = -(-num_kb // ks) if ks > 1 else num_kb
            uneven += 2 <= ks <= 4 and per * ks != num_kb
        d = case.operands(F, n, k, m, rank)
        w = _w64(d["packed"], d["qs"], c_oracle)

        def out(name, cols):
            return torch.from_numpy(got[f"{key}_{name}"]).view(BF16).view(m, cols)

        base = d["x"].double() @ w.t() + d["bias"].double()
        _check(out("fwd", n), base)
        _check(out("fwd_lora", n), base + d["u"].double() @ d["v"].double().t())
        _check(out("dx_lora", k), d["dy"].double() @ w + d["g"].double() @ d["a"].double())
    assert uneven >= 3, uneven


@pytest.mark.parametrize("variant", ["f16_compute", "f16_state_f16_out"])
def test_split_k_half_precision_variants(F, c_oracle, variant):
    """fp16 compute over an fp16 state (weights fp16_rn(LUT[j] absmax), one fp16 rounding), and bf16 compute over an fp16
    state with an fp16 output (weights bf16_rn(fp16_rn(LUT[j] absmax)), the bf16 result rounded to fp16: the reduce's
    kOutF16 branch), split-K at a ragged shape: forward with LoRA and bias, dX with LoRA."""
    n, k = 4104, 4160
    m = _tokens_for("splitk", n, k)
    f16 = variant == "f16_compute"
    cdt = H16 if f16 else BF16
    packed, qs = _quant(F, n, k, seed=7, nested=True, state_dtype=H16)
    w = _restated_weight(c_oracle, packed, qs, "fp16")
    w = torch.from_numpy(w if f16 else o.bf16_round(w)).cuda().double()
    x, dy = make_act(m, k, seed=1).to(cdt), make_act(m, n, seed=2).to(cdt)
    bias = make_weight(1, n, seed=3, scale=0.5).view(-1).to(cdt)
    u, v = make_act(m, 56, seed=4).to(cdt), make_weight(n, 56, seed=5, scale=0.05).to(cdt)
    g, a = make_act(m, 136, seed=6).to(cdt), make_weight(136, k, seed=7, scale=0.05).to(cdt)
    rounding = H16 if f16 else BF16
    y = F.nf4_linear_fwd_lora(x, packed, qs, u, v, bias, out_dtype=H16)
    assert y.dtype == H16
    _check(y, x.double() @ w.t() + bias.double() + u.double() @ v.double().t(), rounding)
    dx = F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a, out_dtype=H16)
    assert dx.dtype == H16
    _check(dx, dy.double() @ w + g.double() @ a.double(), rounding)


# ---- 2. grouped launches on the range schedule ------------------------------------------------------------------------

@pytest.mark.parametrize("nprob,n,k", [(3, 4104, 4160), (2, 11000, 1088)], ids=["qkv", "gate_up"])
def test_grouped_range_schedule_matches_oracle(F, c_oracle, nprob, n, k):
    """q/k/v and gate/up with LoRA: U (and G) column slices of one buffer, the forward outputs side by side in one buffer with
    8 sentinel columns after each (a unit that runs from problem p's partial last feature block into problem p + 1 must
    keep their features apart), and the dX sum of the problems in one output."""
    ps, qss = zip(*[_quant(F, n, k, seed=31 * i + n) for i in range(nprob)])
    ws = [_w64(p, qs, c_oracle) for p, qs in zip(ps, qss)]
    sentinel = -12345.0
    for j, m in enumerate([17, 129, 777, 1535]):
        assert 16 < m < SCRATCH_MIN_M and _lib().qb200_nf4_linear_scratch_size(nprob, m, n, k, 0) == 0
        r = RANKS[(2 * j + 1) % len(RANKS)]
        x = make_act(m, k, seed=m)
        ubuf = make_act(m, nprob * r, seed=m + 1)
        us = [ubuf[:, i * r:(i + 1) * r] for i in range(nprob)]
        vs = [make_weight(n, r, seed=m + 2 + i, scale=0.05) for i in range(nprob)]
        pitch = n + 8
        ybuf = torch.full((m, nprob * pitch), sentinel, dtype=BF16, device="cuda")
        ys = F.nf4_linear_group(False, [x] * nprob, list(ps), list(qss), us=us, vs=vs,
                                outs=[ybuf[:, i * pitch:i * pitch + n] for i in range(nprob)])
        for i, y in enumerate(ys):
            _check(y, x.double() @ ws[i].t() + us[i].double() @ vs[i].double().t())
            assert bool((ybuf[:, i * pitch + n:(i + 1) * pitch] == sentinel).all()), (m, i)
        dys = [make_act(m, n, seed=m + 10 + i) for i in range(nprob)]
        gbuf = make_act(m, nprob * r, seed=m + 20)
        gs = [gbuf[:, i * r:(i + 1) * r] for i in range(nprob)]
        as_ = [make_weight(r, k, seed=m + 30 + i, scale=0.05) for i in range(nprob)]
        dx = F.nf4_linear_group(True, dys, list(ps), list(qss), us=gs, vs=as_)
        _check(dx, sum(dy.double() @ w + g.double() @ a.double() for dy, w, g, a in zip(dys, ws, gs, as_)))


# ---- 3. reads stay inside each operand ---------------------------------------------------------------------------------

@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "row_scaled"])
@pytest.mark.parametrize("schedule", ["splitk", "range"])
def test_reads_stay_inside_each_operand(F, schedule, scaled):
    """Forward (bias, LoRA) and dX (LoRA) over a plain state at 4104 x 4160, r = 24, with NaN where a correct kernel never
    reads: activations with a row pitch past C (and rows past T), U with a pitch past r, V as the prefix of a NaN-filled
    allocation, the fp32 absmax and the row scales each followed by NaN, the packed weight followed by 0xFF bytes.  A dX
    that read weight rows past N would multiply NaN weights by the activation's zero fill.  Every output is finite and
    bitwise the unpadded call's."""
    n, k, r = 4104, 4160, 24
    m = _tokens_for(schedule, n, k)
    packed, qs = _quant(F, n, k, seed=51, nested=False)
    packed = packed.contiguous()
    scale = (torch.rand(n, generator=torch.Generator().manual_seed(52)) + 0.5).cuda()
    scales, pscales = ([scale], [_prefix(scale, float("nan"))]) if scaled else (None, None)
    pqs = F.QuantState(absmax=_prefix(qs.absmax, float("nan")), shape=qs.shape, code=qs.code, blocksize=64, quant_type="nf4",
                       dtype=qs.dtype)
    ppacked = _prefix(packed, 0xFF)
    x, dy = make_act(m, k, seed=53), make_act(m, n, seed=54)
    bias = make_weight(1, n, seed=55, scale=0.5).view(-1)
    u, g = make_act(m, r, seed=56), make_act(m, r, seed=57)
    v, a = make_weight(n, r, seed=58, scale=0.05), make_weight(r, k, seed=59, scale=0.05)
    for is_bwd, inp, lu, lv, b in ((False, x, u, v, [bias]), (True, dy, g, a, None)):
        ref = F.nf4_linear_group(is_bwd, [inp], [packed], [qs], b, [lu], [lv], row_scales=scales)
        got = F.nf4_linear_group(is_bwd, [_padded(inp)], [ppacked], [pqs], b, [_padded(lu)], [_prefix(lv, float("nan"))],
                                 row_scales=pscales)
        ref, got = (ref, got) if is_bwd else (ref[0], got[0])
        torch.cuda.synchronize()
        assert bool(torch.isfinite(got).all()) and torch.equal(got, ref), is_bwd


# ---- 4. pitched and offset outputs -------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def kernel_names(tmp_path_factory):
    """The kernels each call of test_pitched_and_offset_outputs launches, recorded by fused_kernel_names_case.py in a process
    of its own."""
    path = tmp_path_factory.mktemp("kernel_names") / "names.json"
    ms = [str(_tokens_for(s, names_case.N, names_case.K)) for s in ("splitk", "range")]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "fused_kernel_names_case.py"), str(path), *ms],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    with open(path) as f:
        return json.load(f)


@pytest.mark.parametrize("dname", list(names_case.DTYPES))
@pytest.mark.parametrize("is_bwd", [False, True], ids=["fwd", "dx"])
@pytest.mark.parametrize("schedule", ["splitk", "range"])
def test_pitched_and_offset_outputs(F, kernel_names, schedule, is_bwd, dname):
    """Each output a [T, F] view, at an element offset of 0, 1, 2, 4 or 8 and a row pitch of F, F + 4 or F + 8, of a flat
    sentinel-filled buffer (bf16 compute; an fp16 output is the bf16 result rounded to fp16).  Every element outside the view
    keeps its sentinel.  A view whose base the split-K reduce's vector stores can reach (8-byte aligned for a 16-bit output,
    16-byte for fp32) gets bitwise the dense call's output; any other runs un-split, with no reduce launch, and gets bitwise
    the output of the same call given no workspace."""
    out_dtype = names_case.DTYPES[dname]
    m = _tokens_for(schedule, names_case.N, names_case.K)
    f_out = names_case.K if is_bwd else names_case.N
    ops = names_case.operands(F, m, is_bwd)
    packed, qs, inp, bias = ops
    dense = names_case.call(F, ops, is_bwd, out_dtype)
    unsplit = _group_ex(F, is_bwd, inp, packed, qs, torch.empty_like(dense), None, out_dtype=out_dtype, bias=bias)
    if schedule == "splitk":
        assert not torch.equal(dense, unsplit)   # the split sum rounds differently somewhere: the comparisons below tell
    names = kernel_names[names_case.key(schedule, is_bwd, dname)]
    assert any("splitk_reduce" in s for s in names) == (schedule == "splitk"), names
    sentinel = torch.tensor(names_case.SENTINEL, dtype=out_dtype).item()
    align = 16 if out_dtype == F32 else 8
    for pad in names_case.PITCH_PADS:
        for off in names_case.OFFSETS:
            what = (pad, off)
            buf, out = names_case.view(m, f_out, pad, off, out_dtype)
            assert names_case.call(F, ops, is_bwd, out_dtype, out).data_ptr() == out.data_ptr()
            k = names_case.key(schedule, is_bwd, dname, pad, off)
            assert kernel_names[k + "-base16"] == out.data_ptr() % 16, what
            names = kernel_names[k]
            assert any("nf4_gemm_wgmma_kernel" in s for s in names), (what, names)
            if schedule == "splitk" and out.data_ptr() % align != 0:
                assert not any("splitk_reduce" in s for s in names), (what, names)
                assert torch.equal(out, unsplit), what
            else:
                assert any("splitk_reduce" in s for s in names) == (schedule == "splitk"), (what, names)
                assert torch.equal(out, dense), what
            inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
            inside[off:off + m * (f_out + pad)].view(m, f_out + pad)[:, :f_out] = True
            assert bool((buf[~inside] == sentinel).all()), what


# ---- 5. row scales at non-power-of-two values --------------------------------------------------------------------------

def _row_scale(n, seed):
    """Per-row scales around 0.7, 1.3, 3.1 and -0.45, none a power of two."""
    gen = torch.Generator().manual_seed(seed)
    base = torch.tensor([0.7, 1.3, 3.1, -0.45])[torch.randint(0, 4, (n,), generator=gen)]
    return (base * (1.0 + 0.1 * torch.rand(n, generator=gen))).cuda()


def _scaled_case(F, c_oracle, nested, compute, n=1000, k=1088):
    cdt = H16 if compute == "f16" else BF16
    packed, qs = _quant(F, n, k, seed=71, nested=nested, state_dtype=cdt)
    s = _row_scale(n, seed=72)
    w = _restated_weight(c_oracle, packed, qs, "fp16" if compute == "f16" else "bf16", s)
    return cdt, packed, qs, s, w


def _identity_slices(size, m):
    """Row offsets of m-row slices of eye(size) that cover every row (the last slice overlaps the one before it)."""
    return sorted({min(j, size - m) for j in range(0, size, m)})


@pytest.mark.parametrize("compute", ["bf16", "f16"])
@pytest.mark.parametrize("nested", [True, False], ids=["nested", "plain"])
@pytest.mark.parametrize("kernel", ["skinny", "splitk", "range"])
def test_row_scale_folds_into_absmax_exactly(F, c_oracle, kernel, nested, compute):
    """Row scales varying per row at non-power-of-two values, on a ragged shape (1000 x 1088): slices of the identity make
    every output one product 1.0 * w, so the forward gives rows of diag(s) W transposed and dX rows of diag(s) W, bit for
    bit as the oracle restates them: 16-bit_rn(LUT[j] * fl32(absmax * s)), up to the sign of zeros (a negative scale makes
    the table's zero -0, which the accumulator turns into +0).  A scale applied to the rounded weight or to the output
    rounds differently."""
    n, k = 1000, 1088
    cdt, packed, qs, s, w = _scaled_case(F, c_oracle, nested, compute, n, k)
    m = 16 if kernel == "skinny" else _tokens_for(kernel, n, k)
    assert _schedule(m, n, k, False) == kernel
    eye_k, eye_n = torch.eye(k, dtype=cdt, device="cuda"), torch.eye(n, dtype=cdt, device="cuda")
    for j in _identity_slices(k, m):
        y = F.nf4_linear_group(False, [eye_k[j:j + m]], [packed], [qs], row_scales=[s])[0]
        assert np.array_equal(y.float().cpu().numpy(), w[:, j:j + m].T), j
    if kernel == "skinny":
        return
    assert _schedule(m, n, k, True) == kernel
    for j in _identity_slices(n, m):
        dx = F.nf4_linear_group(True, [eye_n[j:j + m]], [packed], [qs], row_scales=[s])
        assert np.array_equal(dx.float().cpu().numpy(), w[j:j + m]), j


@pytest.mark.parametrize("kernel", ["skinny", "splitk", "range"])
def test_row_scaled_random_inputs_match_float64(F, c_oracle, kernel):
    """Random activations through the row-scaled weights of a nested state: forward and dX against float64."""
    n, k = 1000, 1088
    _, packed, qs, s, w = _scaled_case(F, c_oracle, True, "bf16", n, k)
    w = torch.from_numpy(w).cuda().double()
    m = 16 if kernel == "skinny" else _tokens_for(kernel, n, k)
    assert _schedule(m, n, k, False) == kernel
    x = make_act(m, k, seed=73)
    _check(F.nf4_linear_group(False, [x], [packed], [qs], row_scales=[s])[0], x.double() @ w.t())
    if kernel != "skinny":
        assert _schedule(m, n, k, True) == kernel
        dy = make_act(m, n, seed=74)
        _check(F.nf4_linear_group(True, [dy], [packed], [qs], row_scales=[s]), dy.double() @ w)


# ---- 6. ordering without host syncs ------------------------------------------------------------------------------------

def _chain(F, ws):
    """Four calls of `qb200_nf4_linear_ex` through the one workspace `ws`, each reading what an earlier one wrote: split-K
    forwards of two weights on one input, a split-K dX whose input is the first forward's output, and a range-schedule
    forward of a third weight whose input is that dX's output.  Returns (the number of calls, run(i, inputs) -> output)."""
    n, k, n2 = 4104, 4160, 11000
    m = _tokens_for("splitk", n, k)
    assert _schedule(m, n2, k, False) == "range"
    weights = [_quant(F, n, k, seed=81), _quant(F, n, k, seed=82), _quant(F, n2, k, seed=83)]
    weights = [(p.contiguous(), qs) for p, qs in weights]
    # (is_bwd, weight, input: the call whose output it reads, or -1 for x)
    calls = [(False, 0, -1), (False, 1, -1), (True, 0, 0), (False, 2, 2)]
    x = make_act(m, k, seed=84)

    def run(i, outs):
        is_bwd, wi, src = calls[i]
        packed, qs = weights[wi]
        inp = x if src < 0 else outs[src]
        n_w, k_w = qs.shape
        out = torch.empty((m, k_w if is_bwd else n_w), dtype=BF16, device="cuda")
        rc = _lib().qb200_nf4_linear_ex(int(is_bwd), inp.data_ptr(), packed.data_ptr(), *_state_ptrs(F, qs), None, None, None, 0,
                                        out.data_ptr(), m, n_w, k_w, ws.data_ptr(), ws.numel(), F.stream_ptr(inp.device))
        assert rc == 0, _lib().qb200_last_error()
        return out

    for is_bwd, wi, _ in calls[:3]:
        assert _schedule(m, *weights[wi][1].shape, is_bwd) == "splitk"
    return len(calls), run


def _synced(ncalls, run):
    outs = []
    for i in range(ncalls):
        torch.cuda.synchronize()
        outs.append(run(i, outs))
        torch.cuda.synchronize()
    return outs


def _workspace_for_chain():
    return torch.empty(max(_workspace(m, 4104, 4160, d) for m in TOKENS for d in (False, True)), dtype=torch.uint8, device="cuda")


def test_split_k_chain_without_syncs(F):
    """Each output of the unsynchronized chain is bitwise that of the chain run with a sync around every call: a GEMM that
    wrote its partials while the previous reduce still read them, or a launch that read a reduce's output before it was
    stored, would differ."""
    ws = _workspace_for_chain()
    ncalls, run = _chain(F, ws)
    torch.cuda.synchronize()
    got = []
    for i in range(ncalls):
        got.append(run(i, got))
    ref = _synced(ncalls, run)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), i


def test_split_k_chain_replays_under_cuda_graphs(F):
    """The same chain captured in one CUDA graph and replayed once."""
    ws = _workspace_for_chain()
    ncalls, run = _chain(F, ws)
    ref = _synced(ncalls, run)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up: tensor maps, kernel attributes, schedules
        warm = []
        for i in range(ncalls):
            warm.append(run(i, warm))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = []
        for i in range(ncalls):
            static.append(run(i, static))
    for t in static:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(static, ref)):
        assert torch.equal(a, b), i
