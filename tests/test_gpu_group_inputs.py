"""Grouped NF4 forwards whose problems read different inputs, against float64.

A grouped forward takes one input per problem, each with its own pointer and row pitch, and every kernel picks the
activation map of the problem a unit belongs to.  QDoRA with dropout relies on that (q/k/v and gate/up each see their own
dropout mask: Q = group(x_lora_p, U_p, B_p) and P = group(x - x_lora_p)), as does DoRA's grouped weight norm (the adapters
A_p as r-token inputs).  A kernel, schedule or plan that read problem 0's input or pitch for every problem, or decoded the
wrong problem for its activations while using the right one for its weights, would pass a test that gives every problem
the same tensor; every check here gives each problem its own, and every parity check has a negative control: the float64
reference that feeds problem 0's input to every problem misses the bar.

1. The grouped call at the kernel level: each path (the skinny kernels, the 1-token kernel, the fused kernel's range
   schedule, the scratch path) with each variant (nested and plain states, LoRA at r = 16 and 136, a bias, row scales with
   one problem unscaled, fp32 and fp16 outputs, fp16 compute, bf16 compute over an fp16 state), inputs of different
   pitches and offsets; bit for bit against contiguous copies, the single-problem calls and a permutation of the problems.
2. DoRA's grouped weight norm against the float64 norm of W + s B A.
3. QDoRA's grouped step with dropout at training token counts against a float64 restatement of peft's DoraLinearLayer.
4. torch.library.opcheck of `qlora_b200::nf4_linear_group` with distinct, pitched inputs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import group_inputs_case as case
from fp16_helpers import assert_close_f16, f16_round, np32
from gpu_helpers import make_act, make_weight, rel_err
from oracle import nf4_oracle as o
from test_gpu_dora import _dora_ref
from test_gpu_fused_edges import _check, _padded, _restated_weight, _w64

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, H16, F32 = torch.bfloat16, torch.float16, torch.float32
SCRATCH_MIN_M = 1536


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    return F


def _lib():
    from qlora_b200 import _lib

    return _lib.load()


# ---- 1. distinct inputs at the kernel level ----------------------------------------------------------------------------

def _expected_path(variant, m):
    """The path a grouped forward of `variant` takes at m tokens: the skinny kernels up to 16 tokens with a 16-bit output,
    the scratch path from SCRATCH_MIN_M tokens under bf16 compute over a bf16 state with a bf16 or fp32 output and no row
    scales, else the fused kernel's range schedule (a grouped call never splits K)."""
    cdt, sdt, out = case.dtypes(variant)
    if m <= 16 and out != F32:
        return "skinny1" if m == 1 else "skinny"
    if m >= SCRATCH_MIN_M and cdt == BF16 and sdt != H16 and out != H16 and variant != "row_scales":
        return "scratch"
    return "range"


def test_token_counts_reach_every_path():
    """The cases reach the 1-token kernel, the skinny kernels, the range schedule and the scratch path; each variant runs at
    a token count of every class, and each token count and shape is used.  The size queries agree: no workspace at the
    skinny counts, and a scratch from SCRATCH_MIN_M tokens on."""
    lib = _lib()
    paths = {_expected_path(v, m) for v, m, _ in case.CASES}
    assert paths == {"skinny1", "skinny", "range", "scratch"}, paths
    for variant in case.VARIANTS:
        ms = {m for v, m, _ in case.CASES if v == variant}
        assert all(any(m in ms for m in cls) for cls in case.TOKENS.values()), (variant, ms)
    assert {m for _, m, _ in case.CASES} == {m for cls in case.TOKENS.values() for m in cls}
    assert {s for _, _, s in case.CASES} == set(case.SHAPES)
    for variant, m, shape in case.CASES:
        n, k, nprob = case.SHAPES[shape]
        if m <= 16:
            assert lib.qb200_nf4_linear_workspace_size(m, n, k, 0) == 0
        assert (lib.qb200_nf4_linear_scratch_size(nprob, m, n, k, 0) > 0) == (m >= SCRATCH_MIN_M), (m, shape)
        if _expected_path(variant, m) == "scratch":
            assert lib.qb200_nf4_linear_scratch_size(1, m, n, k, 0) > 0


@pytest.fixture(scope="module")
def recorded(tmp_path_factory):
    """group_inputs_case.py's record (kernel names of every grouped call, single-problem outputs), in a process with split-K
    off."""
    path = tmp_path_factory.mktemp("group_inputs") / "record.npz"
    env = dict(os.environ, QB200_SPLITK_MAX_T="0")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "group_inputs_case.py"), str(path)],
                       capture_output=True, text=True, env=env, timeout=1500)
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(path)


_REF_W = {}


def _oracle_w64(c_oracle, packed, qs, table="bf16"):
    """The weight [N, K] as the kernels read it, float64 on the GPU, cached per packed weight: the C oracle's bf16 weight
    ('bf16'), the fp16 table ('fp16': fp16 compute over an fp16 state) or the fp16 table rounded to bf16 ('bf16_of_fp16':
    bf16 compute over an fp16 state)."""
    key = (packed.data_ptr(), table)
    if key not in _REF_W:
        if table == "bf16":
            _REF_W[key] = _w64(packed, qs, c_oracle)
        else:
            w = _restated_weight(c_oracle, packed, qs, "fp16")
            _REF_W[key] = torch.from_numpy(w if table == "fp16" else o.bf16_round(w)).cuda().double()
    return _REF_W[key]


def _ref_weight(c_oracle, d, i):
    """Problem i's weight as the kernels read it (with a row scale: the bf16 table of the row-scaled absmax)."""
    packed, qs = d["packeds"][i], d["states"][i]
    scale = None if d["scales"] is None else d["scales"][i]
    if scale is not None:
        return torch.from_numpy(_restated_weight(c_oracle, packed, qs, "bf16", scale)).cuda().double()
    table = "bf16" if d["sdt"] != H16 else ("fp16" if d["cdt"] == H16 else "bf16_of_fp16")
    return _oracle_w64(c_oracle, packed, qs, table)


def _reference(d, ws, i, x):
    """Problem i's output in float64 for the input x."""
    ref = x.double() @ ws[i].t()
    if d["biases"] is not None:
        ref += d["biases"][i].double()
    if d["us"] is not None:
        ref += d["us"][i].double() @ d["vs"][i].double().t()
    return ref


def _parity(y, ref64, cdt):
    """The parity bar: assert_close_bf16 at 1e-3 against the reference rounded once (bf16, then the output dtype), or
    assert_close_f16 against the fp16-rounded reference under fp16 compute."""
    if cdt == H16:
        assert_close_f16(np32(y), f16_round(ref64.float().cpu().numpy()))
    else:
        _check(y, ref64)


def _misses(y, ref64, cdt):
    try:
        _parity(y, ref64, cdt)
    except AssertionError:
        return True
    return False


def _pitched(xs):
    """Problem 0's input as it is, problem 1's as columns [64, 64 + C) of a NaN-filled [T, C + 136] buffer, problem 2's as
    rows [24, 24 + T) of a NaN-filled [T + 40, C + 8] buffer: three row pitches and three base offsets."""
    out = [xs[0]]
    m, c = xs[1].shape
    buf = torch.full((m, c + 136), float("nan"), dtype=xs[1].dtype, device="cuda")
    buf[:, 64:64 + c] = xs[1]
    out.append(buf[:, 64:64 + c])
    if len(xs) > 2:
        rows = _padded(torch.cat([torch.zeros(24, c, dtype=xs[2].dtype, device="cuda"), xs[2]]), extra_rows=16, extra_cols=8)
        rows[:24] = float("nan")
        out.append(rows[24:])
    for t in out:   # the kernels read these views in place (16-byte aligned, pitch a multiple of 8)
        assert t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0
    assert len({t.stride(0) for t in out}) == len(out)
    return out


@pytest.mark.parametrize("cs", case.CASES, ids=[case.case_id(c) for c in case.CASES])
def test_grouped_inputs_match_float64(F, c_oracle, recorded, cs):
    """The grouped forward with its own input per problem, given as views of different pitches and offsets: the path the
    kernel names show; every output finite and bitwise that of the call on contiguous copies and of the single-problem call
    on its own operands (the same kernel, split-K off); permuting the problems permutes the outputs exactly; each output
    within the parity bar of float64, which the reference that feeds problem 0's input to every problem misses."""
    variant, m, shape = cs
    cid = case.case_id(cs)
    want = _expected_path(variant, m)
    assert case.path(recorded[f"{cid}__names"]) == want, list(recorded[f"{cid}__names"])
    d = case.operands(F, cs)
    nprob, cdt = d["nprob"], d["cdt"]
    xs = _pitched(d["xs"])
    ys = case.call(F, d, xs=xs)
    dense = case.call(F, d)
    torch.cuda.synchronize()
    for i, (y, yd) in enumerate(zip(ys, dense)):
        assert y.dtype == d["out_dtype"] and bool(torch.isfinite(y).all()) and torch.equal(y, yd), i
        assert case.path(recorded[f"{cid}__single{i}_names"]) == want, i
        assert np.array_equal(case.bits(y), recorded[f"{cid}__single{i}"]), i
    order = [1, 0] if nprob == 2 else [2, 0, 1]
    for j, y in enumerate(case.call(F, d, xs=xs, order=order)):
        assert torch.equal(y, ys[order[j]]), (j, order)
    ws = [_ref_weight(c_oracle, d, i) for i in range(nprob)]
    for i, y in enumerate(ys):
        _parity(y, _reference(d, ws, i, d["xs"][i]), cdt)
        if i > 0:
            assert _misses(y, _reference(d, ws, i, d["xs"][0]), cdt), i


# ---- 2. DoRA's grouped weight norm -------------------------------------------------------------------------------------

@pytest.mark.parametrize("r", [8, 16, 64, 136, 256])
@pytest.mark.parametrize("n,k", [(4096, 4096), (11008, 4096)], ids=["4096x4096", "11008x4096"])
def test_grouped_dora_weight_norm_matches_float64(F, c_oracle, n, k, r):
    """`dora_weight_norm` over three weights with their own adapters: every row within 2^-8 relative of the float64 norm of
    W_oracle + s B A, for ||s B A||_F = 1 % and 50 % of ||W||_F.  P = A_p . W_p^T comes from one grouped forward with the
    adapters as r-token inputs and an fp32 output, on the fused kernel's range schedule at every rank (an fp32 output never
    takes the skinny kernels, and grouped calls never split K); for r <= 16 the single-problem call takes that schedule too
    (no split-K workspace up to 16 tokens), so its norms are the grouped ones bit for bit.  At 50 % the reference whose P
    reads A_0 for every problem misses the bar (at 1 % the adapter moves the norm by less than the bar)."""
    lib = _lib()
    assert lib.qb200_nf4_linear_scratch_size(3, r, n, k, 0) == 0
    ps, qss = case.weights(F, n, k, 3, True, BF16)
    ws = [_oracle_w64(c_oracle, p, qs) for p, qs in zip(ps, qss)]
    s = 16.0 / r
    for ratio in (0.01, 0.5):
        as_ = [make_weight(r, k, seed=r + 10 * i, scale=0.05) for i in range(3)]
        bs = []
        for i in range(3):
            b = make_weight(n, r, seed=r + 10 * i + 1, scale=0.05)
            ba = b.double() @ as_[i].double()
            bs.append((b.double() * (ratio * ws[i].norm() / (s * ba.norm()))).to(BF16))   # ||s B A|| = ratio ||W||
        norms = F.dora_weight_norm(ps, qss, as_, bs, s)
        for i in range(3):
            a64, b64 = as_[i].double(), bs[i].double()
            ref = torch.linalg.norm(ws[i] + s * (b64 @ a64), dim=1)
            assert norms[i].shape == (n,) and norms[i].dtype == F32
            err = ((norms[i].double() - ref).abs() / ref).max().item()
            assert err <= 2.0 ** -8, (ratio, i, err)
            if r <= 16:
                assert torch.equal(norms[i], F.dora_weight_norm(ps[i], qss[i], as_[i], bs[i], s)), (ratio, i)
            if ratio == 0.5 and i > 0:   # n^2 = ||W||^2 + 2 s sum_j B[f, j] P[j, f] + s^2 (B A A^T B^T)_ff with P read from A_0
                cross = lambda a: (b64 * (a.double() @ ws[i].t()).t()).sum(1)   # noqa: E731
                bad = (ref * ref - 2 * s * cross(as_[i]) + 2 * s * cross(as_[0])).clamp_min(0).sqrt()
                bad_err = ((norms[i].double() - bad).abs() / bad).max().item()
                assert bad_err > 2.0 ** -8, (i, bad_err)


# ---- 3. QDoRA's grouped step with dropout at training token counts -----------------------------------------------------

DORA_SHAPES = {"qkv": (4096, 4096, 3), "gate_up": (11008, 4096, 2)}
# (tokens, dropout): the fused kernel at 300 tokens; at 1543 and 2048 the unscaled launches take the scratch path
DORA_STEPS = [(300, True), (1543, True), (2048, True), (2048, False)]
DORA_CASES = [(g, r, m, p) for g in DORA_SHAPES for r in (64, 136) for m, p in DORA_STEPS]
NAMES = ("y", "dx", "dA", "dB", "dm")
CEIL = 5e-3   # the bar where twice the peft form's error is lower (the fused path measures up to 3.3e-3)


def _base(q, n_in, n_out):
    """A Linear4bit over a bf16 weight (a bf16 quant state: the fused DoRA path)."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF16)
    try:
        base = q.nn.Linear4bit(n_in, n_out, bias=False, compute_dtype=BF16, quant_type="nf4").cuda()
    finally:
        torch.set_default_dtype(prev)
    assert base.weight.quant_state.dtype == BF16
    return base


def _grads(ys, gys, leaves):
    torch.autograd.backward(ys, gys)
    return [t.grad for t in leaves]


def dora_step_errors(q, c_oracle, group, r, m, dropout, record=None):
    """One grouped QDoRA forward and backward: the fused path (`dora_linear4bit_group`) and peft's form on the library's
    unfused kernels (`dora_linear4bit_peft` per linear), both against the float64 restatement on the oracle's weights with
    the same masks.  Returns {quantity: [(fused error, peft-form error) of each problem]} (relative Frobenius), and the negative
    controls {name: error of the fused result against a wrong reference}.  `record`, when given, collects the grouped calls
    of the fused path as (is_bwd, problems, tokens, row-scaled, left its weights in a scratch)."""
    F = q.functional
    n_out, n_in, nprob = DORA_SHAPES[group]
    s = 16.0 / r
    torch.manual_seed(1000 * r + m)
    bases = [_base(q, n_in, n_out) for _ in range(nprob)]
    ws = [_w64(b.weight.data, b.weight.quant_state, c_oracle) for b in bases]
    As = [(torch.randn(r, n_in, device="cuda") * 0.05).to(BF16) for _ in range(nprob)]
    Bs = [(torch.randn(n_out, r, device="cuda") * 0.02).to(BF16) for _ in range(nprob)]
    Ms = [(w.norm(dim=1) * (1 + 0.1 * torch.randn(n_out, device="cuda", dtype=torch.float64))).to(BF16) for w in ws]
    x = make_act(m, n_in, seed=m + r)
    gys = [make_act(m, n_out, seed=m + r + 1 + i) for i in range(nprob)]
    masks = [((torch.rand(m, n_in, device="cuda") >= 0.1).float() / 0.9).to(BF16) for _ in range(nprob)] if dropout else None

    def leaves():
        return [x.detach().clone().requires_grad_(True)], [[t.detach().clone().requires_grad_(True) for t in ts] for ts in (As, Bs, Ms)]

    (xf,), (Af, Bf, Mf) = leaves()
    xls = [xf * mk for mk in masks] if dropout else None
    assert q.lora._dora_fusable(xf, bases, Af, Bf, Mf, xls)
    orig = F.nf4_linear_group

    def recording(is_bwd, inputs, *args, **kw):
        res, scratch = orig(is_bwd, inputs, *args, return_scratch=True, **kw)
        record.append((is_bwd, len(inputs), inputs[0].shape[0], kw.get("row_scales") is not None, scratch is not None))
        return res

    if record is not None:
        F.nf4_linear_group = recording
    try:
        ys = list(q.dora_linear4bit_group(xf, bases, Af, Bf, Mf, s, xls))
        fused = [y.detach() for y in ys] + _grads(ys, gys, [xf] + Af + Bf + Mf)
    finally:
        F.nf4_linear_group = orig

    (xp,), (Ap, Bp, Mp) = leaves()
    ys = [q.lora.dora_linear4bit_peft(xp, bases[i], Ap[i], Bp[i], Mp[i], s, xp * masks[i] if dropout else None)
          for i in range(nprob)]
    peft = [y.detach() for y in ys] + _grads(ys, gys, [xp] + Ap + Bp + Mp)

    def reference(mask_of):
        x64 = x.double().requires_grad_(True)
        A64, B64, M64 = ([t.double().requires_grad_(True) for t in ts] for ts in (As, Bs, Ms))
        ys = [_dora_ref(x64, x64 * masks[mask_of(i)].double() if dropout else None, ws[i], A64[i], B64[i], M64[i], s)
              for i in range(nprob)]
        ref = [y.detach() for y in ys] + _grads(ys, [g.double() for g in gys], [x64] + A64 + B64 + M64)
        cs = [(M64[i].detach() / torch.linalg.norm(ws[i] + s * (B64[i].detach() @ A64[i].detach()), dim=1)) for i in range(nprob)]
        return ref, cs

    ref, cs = reference(lambda i: i)

    def split(vals):   # [y_0.., dx, dA_0.., dB_0.., dm_0..] -> {quantity: [per problem]}
        return {"y": vals[:nprob], "dx": [vals[nprob]] * nprob, "dA": vals[nprob + 1:2 * nprob + 1],
                "dB": vals[2 * nprob + 1:3 * nprob + 1], "dm": vals[3 * nprob + 1:]}

    fu, pe, rf = split(fused), split(peft), split(ref)

    def err(a, b):
        return rel_err(a.detach().double().cpu().numpy(), b.detach().double().cpu().numpy())

    errors = {name: [(err(fu[name][i], rf[name][i]), err(pe[name][i], rf[name][i])) for i in range(nprob)] for name in NAMES}
    # dm = sum_t dy * Q / n with dropout, sum_t dy * y / (c n) without: the other form's division is off by c per feature
    controls = {"dm_other_form": [err(fu["dm"][i].double() * (1 / cs[i] if dropout else cs[i]), rf["dm"][i]) for i in range(nprob)]}
    if dropout:   # the reference that gives every linear problem 0's mask
        bad = split(reference(lambda i: 0)[0])
        controls["dm_mask0"] = [err(fu["dm"][i], bad["dm"][i]) for i in range(1, nprob)]
        controls["dA_mask0"] = [err(fu["dA"][i], bad["dA"][i]) for i in range(1, nprob)]
    return errors, controls


def _bar(fused_peft):
    """Twice the peft form's error, or CEIL where that is lower."""
    return max(2 * fused_peft[1], CEIL)


@pytest.mark.parametrize("group,r,m,dropout", DORA_CASES,
                         ids=[f"{g}-r{r}-{m}-{'p0.1' if p else 'p0'}" for g, r, m, p in DORA_CASES])
def test_grouped_dora_step_matches_float64(c_oracle, group, r, m, dropout):
    """y and the gradients of x, A, B and m of `dora_linear4bit_group` with a dropout mask per linear, against float64
    (test_gpu_dora.py's restatement of peft's DoraLinearLayer on the C oracle's weights, the same masks); each within twice
    the error of peft's form on the library's unfused kernels (`dora_linear4bit_peft` per linear), or within CEIL.  The
    grouped launches take the scratch path where the token count asks for it: with dropout the forward's Q and P launches
    and the dX of the base term (unscaled, one input per problem), while every row-scaled launch keeps the fused kernel.

    Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W): relative Frobenius error against float64 over the 16 cases
    and every linear, fused path / peft form (the no-dropout cases at 2048 tokens apart):

        quantity   dropout                          no dropout
        y          2.50e-3..2.53e-3 / 3.65e-3..3.74e-3   2.67e-3..2.69e-3 / 3.55e-3..3.60e-3
        dx         2.85e-3..3.32e-3 / 4.21e-3..4.61e-3   2.67e-3..2.68e-3 / 4.28e-3..4.64e-3
        dA         3.30e-3..3.33e-3 / 4.13e-3..4.50e-3   2.86e-3..2.88e-3 / 3.81e-3..4.18e-3
        dB         3.31e-3..3.33e-3 / 4.14e-3..4.49e-3   2.86e-3..2.89e-3 / 3.81e-3..4.17e-3
        dm         2.79e-3..2.97e-3 / 4.43e-3..4.58e-3   3.12e-3..3.28e-3 / 4.15e-3..4.32e-3

    The bars (twice the peft form's error) are 7.1e-3 to 9.3e-3.  The negative controls miss them by 11x or more: dm in
    the other form's division (by c n instead of n, or the reverse: error 0.095 to 0.116) and, with dropout, dm and dA
    against the reference that gives every linear problem 0's mask (0.44 to 0.48)."""
    import qlora_b200 as q

    calls = []
    errors, controls = dora_step_errors(q, c_oracle, group, r, m, dropout, record=calls)
    nprob = DORA_SHAPES[group][2]
    scratch = m >= SCRATCH_MIN_M
    fwd_multi = [c for c in calls if not c[0] and c[2] == m]
    assert fwd_multi and all(c[1] == nprob for c in fwd_multi), calls
    for is_bwd, _, tokens, scaled, took in calls:
        assert took == (tokens == m and scratch and not scaled), calls
    if dropout:
        assert sum(1 for c in fwd_multi if not c[3]) == 2, calls
    for name, per in errors.items():
        for i, fp in enumerate(per):
            assert fp[0] <= _bar(fp), (name, i, fp)
    for i, e in enumerate(controls["dm_other_form"]):
        assert e >= 5 * _bar(errors["dm"][i]), ("dm_other_form", i, e)
    if dropout:
        for key, name in (("dm_mask0", "dm"), ("dA_mask0", "dA")):
            for i, e in enumerate(controls[key], start=1):
                assert e >= 5 * _bar(errors[name][i]), (key, i, e)


# ---- 4. the custom op's compile contract ------------------------------------------------------------------------------

@pytest.mark.parametrize("m", [5, 300, 2048], ids=["skinny", "range", "scratch"])
def test_opcheck_with_distinct_pitched_inputs(m):
    """`torch.library.opcheck` of `qlora_b200::nf4_linear_group` on three problems with their own inputs, given as views of
    different pitches and offsets, LoRA at r = 16 and a bias."""
    import qlora_b200._ops  # noqa: F401
    from test_gpu_compile import _group_args

    n = k = 1024
    lib = _lib()
    assert (lib.qb200_nf4_linear_scratch_size(3, m, n, k, 0) > 0) == (m >= SCRATCH_MIN_M)
    args = list(_group_args(False, m, n, k, nprob=3, r=16, bias=True))
    args[1] = _pitched(args[1])
    torch.library.opcheck(torch.ops.qlora_b200.nf4_linear_group.default, tuple(args))
