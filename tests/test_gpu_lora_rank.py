"""LoRA ranks 72..256 on the fused path: one 64-wide LoRA contraction step per 64 ranks after the NF4 steps, in the fused
and the scratch kernel, and 64-rank chunks in the skinny kernels' epilogues.  Ranks 72, 136 and 200 end in an 8-wide step
whose other 56 columns are TMA zero-fill.

Checked against the C oracle's weights in float64 (the parity bar of test_gpu_scratch_edges.py), fused against scratch bit for
bit, with NaN where a correct kernel never reads, at the module level against the two-step form and peft's DoRA, and in the
benchmarked training step at r = 128 against its float64 restatement."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fp16_helpers import assert_close_f16, f16_round, np32, oracle_w16
from gpu_helpers import assert_close_bf16, bf16_to_f32_np, make_act, make_weight, oracle_weight, rel_err
from oracle import nf4_oracle as o

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, H16, F32 = torch.bfloat16, torch.float16, torch.float32
TOL = 1e-3
RANKS = [72, 128, 136, 200, 256]


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    return F


def _lib():
    from qlora_b200 import _lib

    return _lib.load()


def _quant(F, n, k, seed, nested=True, state_dtype=BF16):
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=seed, dtype=state_dtype), compress_statistics=nested, quant_type="nf4")
    return packed.t(), qs


def _check(y, ref64):
    assert y.dtype == BF16
    assert_close_bf16(bf16_to_f32_np(y), ref64.float().to(BF16).float().cpu().numpy(), TOL)


# ---- 1. parity with the oracle ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("nested", [True, False], ids=["nested", "plain"])
@pytest.mark.parametrize("n,k", [(1000, 1088), (4096, 4096), (11008, 4096)], ids=["1000x1088", "4096x4096", "11008x4096"])
def test_ranks_match_oracle(F, c_oracle, n, k, nested):
    """Forward with bias and dX at every rank: T = 1000 (fused kernel), 2048 and 1543 (scratch path), and 17, 48, 64 (the
    split-K schedule where the library plans it: always for dX here, and for the forward below 11008 features)."""
    lib = _lib()
    packed, qs = _quant(F, n, k, seed=n + k, nested=nested)
    w = torch.from_numpy(oracle_weight(packed, qs, c_oracle)).cuda().double()
    bias = make_weight(1, n, seed=3, scale=0.5).view(-1)
    for m in (1000, 2048, 1543, 17, 48, 64):
        scratch = m >= 1536
        assert (lib.qb200_nf4_linear_scratch_size(1, m, n, k, 0) > 0) == scratch
        if m < 100:
            assert lib.qb200_nf4_linear_workspace_size(m, n, k, 1) > 0
            assert (lib.qb200_nf4_linear_workspace_size(m, n, k, 0) > 0) == (n != 11008)
        x, dy = make_act(m, k, seed=m), make_act(m, n, seed=m + 1)
        base = x.double() @ w.t() + bias.double()
        for r in RANKS:
            u, v = make_act(m, r, seed=10 + r), make_weight(n, r, seed=20 + r, scale=0.05)
            _check(F.nf4_linear_fwd_lora(x, packed, qs, u, v, bias), base + u.double() @ v.double().t())
        base = dy.double() @ w
        for r in RANKS:
            g, a = make_act(m, r, seed=30 + r), make_weight(r, k, seed=40 + r, scale=0.05)
            _check(F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a), base + g.double() @ a.double())
        del base


# ---- 2. fused and scratch kernels, bit for bit -------------------------------------------------------------------------

def test_fused_and_scratch_paths_are_bitwise_equal(tmp_path):
    """Single problems, q/k/v and gate/up forwards with U slices of one buffer, and their dX sums at r = 128, 200, 256, run
    with the scratch path forced and with the fused kernel forced (split-K off in both)."""
    files = {}
    for side, min_m in (("scratch", "17"), ("fused", str(1 << 30))):
        env = dict(os.environ, QB200_SCRATCH_MIN_M=min_m, QB200_SPLITK_MAX_T="0")
        files[side] = tmp_path / f"{side}.npz"
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "lora_rank_case.py"), str(files[side])],
                           capture_output=True, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
    a, b = np.load(files["scratch"]), np.load(files["fused"])
    assert sorted(a.files) == sorted(b.files) and len(a.files) == 2 * 3 * 2 * 3 * 9
    for key in a.files:
        assert np.array_equal(a[key], b[key]), key


# ---- 3. reads stay inside each operand ---------------------------------------------------------------------------------

def _nan_buffer(rows, cols):
    return torch.full((rows, cols), float("nan"), dtype=BF16, device="cuda")


@pytest.mark.parametrize("m", [1000, 2048], ids=["fused", "scratch"])
@pytest.mark.parametrize("r", [136, 256])
def test_reads_stay_inside_lora_operands(F, m, r):
    """Single and grouped (3), forward and dX, at 1000 x 1088: U and G as column slices of a [T + 256, 3 r + 64] buffer,
    V [N, r] as the first N rows of an [N + 64, r] buffer and the dX operand A [r, K] as the first r rows of an [r + 64, K]
    buffer, NaN everywhere else.  Every output is finite and bitwise that of the unpadded call."""
    n, k = 1000, 1088
    ps, qss = zip(*[_quant(F, n, k, seed=23 * i + k) for i in range(3)])
    x = make_act(m, k, seed=1)
    dys = [make_act(m, n, seed=2 + i) for i in range(3)]
    us = [make_act(m, r, seed=10 + i) for i in range(3)]
    vs = [make_weight(n, r, seed=20 + i, scale=0.05) for i in range(3)]
    gs = [make_act(m, r, seed=30 + i) for i in range(3)]
    as_ = [make_weight(r, k, seed=40 + i, scale=0.05) for i in range(3)]

    def slices(ts):
        buf = _nan_buffer(m + 256, 3 * r + 64)
        for i, t in enumerate(ts):
            buf[:m, i * r:(i + 1) * r] = t
        return [buf[:m, i * r:(i + 1) * r] for i in range(3)]

    def rows(t):
        buf = _nan_buffer(t.shape[0] + 64, t.shape[1])
        buf[:t.shape[0]] = t
        return buf[:t.shape[0]]

    pus, pgs, pvs, pas = slices(us), slices(gs), [rows(v) for v in vs], [rows(a) for a in as_]
    assert all(t.is_contiguous() for t in pvs + pas)
    for p in (1, 3):
        got = F.nf4_linear_group(False, [x] * p, list(ps[:p]), list(qss[:p]), us=pus[:p], vs=pvs[:p])
        ref = F.nf4_linear_group(False, [x] * p, list(ps[:p]), list(qss[:p]), us=us[:p], vs=vs[:p])
        got.append(F.nf4_linear_group(True, dys[:p], list(ps[:p]), list(qss[:p]), us=pgs[:p], vs=pas[:p]))
        ref.append(F.nf4_linear_group(True, dys[:p], list(ps[:p]), list(qss[:p]), us=gs[:p], vs=as_[:p]))
        for a, b in zip(got, ref):
            assert bool(torch.isfinite(a).all()) and torch.equal(a, b)


# ---- 4. skinny kernels and the other dtypes ----------------------------------------------------------------------------

@pytest.mark.parametrize("m", [1, 8, 16])
@pytest.mark.parametrize("r", [128, 256])
@pytest.mark.parametrize("dtype", [BF16, H16], ids=["bf16", "fp16"])
def test_skinny_ranks_match_oracle(F, c_oracle, dtype, r, m):
    """Forward with bias on the skinny kernels (<= 16 tokens; one token has its own kernel), 4096 x 4096."""
    n, k = 4096, 4096
    assert _lib().qb200_nf4_linear_workspace_size(m, n, k, 0) == 0
    packed, qs = _quant(F, n, k, seed=m + r, state_dtype=dtype)
    x = make_act(m, k, seed=m).to(dtype)
    u = make_act(m, r, seed=m + 1).to(dtype)
    v = make_weight(n, r, seed=m + 2, scale=0.05, dtype=dtype)
    bias = make_weight(1, n, seed=m + 3, scale=0.5, dtype=dtype).view(-1)
    y = F.nf4_linear_fwd_lora(x, packed, qs, u, v, bias)
    assert y.dtype == dtype
    if dtype == BF16:
        w = oracle_weight(packed, qs, c_oracle)
        ref = x.double() @ torch.from_numpy(w).cuda().double().t() + u.double() @ v.double().t() + bias.double()
        _check(y, ref)
    else:
        w = oracle_w16(c_oracle, packed, qs)
        ref = np32(x) @ w.T + np32(u) @ np32(v).T + np32(bias)
        assert_close_f16(np32(y), f16_round(ref))


@pytest.mark.parametrize("case", ["fp16_compute", "bf16_over_fp16_state"])
def test_other_dtypes_at_rank_128(F, c_oracle, case):
    """Forward and dX at r = 128, 1000 tokens (fused kernel) over 4096 x 4096: fp16 compute over an fp16 state, and bf16
    compute over an fp16 state (weights bf16_rn(fp16_rn(LUT[j] * absmax)))."""
    n, k, m, r = 4096, 4096, 1000, 128
    cdt = H16 if case == "fp16_compute" else BF16
    packed, qs = _quant(F, n, k, seed=5, state_dtype=H16)
    w = oracle_w16(c_oracle, packed, qs)
    if cdt == BF16:
        w = o.bf16_round(w)
    x, dy = make_act(m, k, seed=1).to(cdt), make_act(m, n, seed=2).to(cdt)
    u, v = make_act(m, r, seed=3).to(cdt), make_weight(n, r, seed=4, scale=0.05, dtype=cdt)
    g, a = make_act(m, r, seed=5).to(cdt), make_weight(r, k, seed=6, scale=0.05, dtype=cdt)
    y = F.nf4_linear_fwd_lora(x, packed, qs, u, v)
    dx = F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a)
    y_ref = np32(x) @ w.T + np32(u) @ np32(v).T
    dx_ref = np32(dy) @ w + np32(g) @ np32(a)
    assert y.dtype == cdt and dx.dtype == cdt
    if cdt == H16:
        assert_close_f16(np32(y), f16_round(y_ref))
        assert_close_f16(np32(dx), f16_round(dx_ref))
    else:
        assert_close_bf16(np32(y), o.bf16_round(y_ref), TOL)
        assert_close_bf16(np32(dx), o.bf16_round(dx_ref), TOL)


# ---- 5. module level ---------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def q():
    import qlora_b200 as q

    return q


def _base(q, n_in, n_out):
    """A Linear4bit over a bf16 weight (a bf16 quant state: the fused LoRA and DoRA paths; an fp32 state keeps the two-step
    form under bf16 compute)."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF16)
    try:
        base = q.nn.Linear4bit(n_in, n_out, bias=False, compute_dtype=BF16, quant_type="nf4").cuda()
    finally:
        torch.set_default_dtype(prev)
    assert base.weight.quant_state.dtype == BF16
    return base


def test_group_fusable_follows_the_rank(q):
    x = torch.zeros(4, 512, dtype=BF16, device="cuda")
    bases = [_base(q, 512, 768) for _ in range(3)]
    for r, want in ((128, True), (256, True), (264, False), (132, False)):
        As = [torch.zeros(r, 512, dtype=BF16, device="cuda") for _ in range(3)]
        Bs = [torch.zeros(768, r, dtype=BF16, device="cuda") for _ in range(3)]
        assert q.lora._group_fusable(x, bases, As, Bs, None) == want, r
        assert q.lora._group_fusable(x, bases[:1], As[:1], Bs[:1], None) == want, r


@pytest.mark.parametrize("tokens", [300, 2048], ids=["fused", "scratch"])
@pytest.mark.parametrize("r", [128, 256])
@pytest.mark.parametrize("group", [1, 3])
def test_fused_lora_autograd_matches_two_step(q, group, r, tokens):
    """`lora_linear4bit` / `lora_linear4bit_group` against peft's two-step form on the same kernels: outputs, dX, dA, dB
    within the 4e-3 of test_gpu_linear.py's fused-vs-two-step test."""
    torch.manual_seed(r + group)
    bases = [_base(q, 512, 768) for _ in range(group)]
    As = [(torch.randn(r, 512, device="cuda") * 0.05).to(BF16).requires_grad_(True) for _ in range(group)]
    Bs = [(torch.randn(768, r, device="cuda") * 0.05).to(BF16).requires_grad_(True) for _ in range(group)]
    x = torch.randn(2, tokens // 2, 512, device="cuda", dtype=BF16, requires_grad=True)
    gys = [torch.randn(2, tokens // 2, 768, device="cuda", dtype=BF16) for _ in range(group)]
    assert q.lora._group_fusable(x, bases, As, Bs, None)
    ys = [q.lora_linear4bit(x, bases[0], As[0], Bs[0], 0.25)] if group == 1 else list(q.lora_linear4bit_group(x, bases, As, Bs, 0.25))
    torch.autograd.backward(ys, gys)
    got = [y.detach().float() for y in ys] + [x.grad.float()] + [t.grad.float() for t in As + Bs]
    x2 = x.detach().clone().requires_grad_(True)
    As2, Bs2 = ([t.detach().clone().requires_grad_(True) for t in ts] for ts in (As, Bs))
    ys2 = [bases[i](x2) + torch.nn.functional.linear(torch.nn.functional.linear(x2, As2[i]), Bs2[i]) * 0.25 for i in range(group)]
    torch.autograd.backward(ys2, gys)
    ref = [y.detach().float() for y in ys2] + [x2.grad.float()] + [t.grad.float() for t in As2 + Bs2]
    names = [f"y{i}" for i in range(group)] + ["dx"] + [f"{p}{i}" for p in "AB" for i in range(group)]
    for name, a_, b_ in zip(names, got, ref):
        e = rel_err(a_.cpu().numpy(), b_.cpu().numpy())
        assert e <= 4e-3, (name, e)


@pytest.mark.parametrize("dropout", [False, True])
def test_qdora_rank_128_matches_peft_form(q, dropout):
    """QDoRA at r = 128 runs fused (row-scaled launches and the weight-norm launch that takes A as a 128-token input) and
    agrees with `dora_linear4bit_peft` within test_gpu_dora.py's 1e-2: y and the gradients of x, A, B and m."""
    torch.manual_seed(11)
    F = q.functional
    r, s = 128, 0.5
    base = _base(q, 512, 768)
    w = F.dequantize_4bit(base.weight.data, base.weight.quant_state).float()
    A = (torch.randn(r, 512, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    B = (torch.randn(768, r, device="cuda") * 0.02).to(BF16).requires_grad_(True)
    M = (w.norm(dim=1) * (1 + 0.1 * torch.randn(768, device="cuda"))).to(BF16).requires_grad_(True)
    x = torch.randn(2, 150, 512, device="cuda", dtype=BF16, requires_grad=True)
    gy = torch.randn(2, 150, 768, device="cuda", dtype=BF16)
    xl = (x.detach() * ((torch.rand_like(x.float()) >= 0.1).float() / 0.9).to(BF16)) if dropout else None
    assert q.lora._dora_fusable(x, [base], [A], [B], [M], None if xl is None else [xl])
    norm = F.dora_weight_norm(base.weight.data.t(), base.weight.quant_state, A, B, s)
    want = torch.linalg.norm(w + s * (B.detach().float() @ A.detach().float()), dim=1)
    assert rel_err(norm.cpu().numpy(), want.cpu().numpy()) <= 1e-3
    y = q.dora_linear4bit(x, base, A, B, M, s, xl)
    y.backward(gy)
    got = [y.detach().float(), x.grad.float(), A.grad.float(), B.grad.float(), M.grad.float()]
    x2, A2, B2, M2 = (t.detach().clone().requires_grad_(True) for t in (x, A, B, M))
    y2 = q.lora.dora_linear4bit_peft(x2, base, A2, B2, M2, s, xl)
    y2.backward(gy)
    ref = [y2.detach().float(), x2.grad.float(), A2.grad.float(), B2.grad.float(), M2.grad.float()]
    for name, a_, b_ in zip(("y", "dx", "dA", "dB", "dm"), got, ref):
        e = rel_err(a_.cpu().numpy(), b_.cpu().numpy())
        assert e <= 1e-2, (name, e)


# ---- 6. the benchmarked training step at r = 128 -----------------------------------------------------------------------

STEP_CASES = {
    "fused_p0": dict(seq=1000, p=0.0, accum=1),
    "fused_p0.1": dict(seq=1000, p=0.1, accum=1),
    "scratch_p0": dict(seq=2048, p=0.0, accum=1),
    "scratch_p0.1": dict(seq=2048, p=0.1, accum=1),
}


@pytest.fixture(scope="module")
def S():
    """test_gpu_bench_step.py's step harness and the Llama-QLoRA harness module."""
    import test_gpu_bench_step as S

    from harness import fused_ops

    fused_ops.build()
    assert fused_ops.available()
    return S


def _rank_128(mp, S, **overrides):
    """bench.py's settings, with the tiny model built at LoRA r = 128 (and `overrides`)."""
    import harness.llama_qlora as H

    orig = H.LlamaQLoRA
    mp.setattr(H, "LlamaQLoRA", lambda *a, **kw: orig(*a, **{**kw, "lora_r": 128, **overrides}))
    S._bench_settings(mp, H, fused=True)
    return H


@pytest.mark.parametrize("case", sorted(STEP_CASES))
def test_rank_128_step_matches_float64(S, c_oracle, deterministic, monkeypatch, case):
    """Loss and the 28 adapter gradients of one step against float64, within test_gpu_bench_step.py's ceilings."""
    cfg = STEP_CASES[case]
    with monkeypatch.context() as mp:
        H = _rank_128(mp, S)
        bs = S.BenchStep(H, cfg)
        assert bs.model.layers[0].q_proj.lora_A.weight.shape[0] == 128
        a0 = S._f64(bs.split(bs.gsync.flat_param.clone()))
        out = bs.step(0)
    ref = bs.reference_model(c_oracle)
    seeds = [s for _, s in out["micro"]]
    ref_losses, ref_grads = S.reference_step(bs, ref, a0, 0, seeds)
    for (loss, _), want in zip(out["micro"], ref_losses):
        assert abs(float(loss) - want) <= S.CEIL_LOSS * abs(want), (float(loss), want)
    errs = S.rel_errors(bs.split(out["grad"]), S._sum(ref_grads))
    assert len(errs) == 28
    for n, e in errs.items():
        assert e is not None and e <= S.ceiling(n), (n, e)


@pytest.mark.parametrize("case", ["fused_p0.1", "scratch_p0.1"])
def test_rank_128_checkpointed_step_equals_plain(S, deterministic, monkeypatch, case):
    """Gradient checkpointing (whose recompute hands its bf16 weight copies to the dX launches on the scratch path) leaves
    the loss and every gradient bit for bit as they are without it."""
    res, salts = [], None
    for ckpt in (True, False):
        with monkeypatch.context() as mp:
            H = _rank_128(mp, S, grad_checkpointing=ckpt)
            bs = S.BenchStep(H, STEP_CASES[case], salts=salts)   # the same dropout masks in both models
            assert bs.model.grad_checkpointing == ckpt
            salts = bs.salts()
            res.append(bs.step(0))
    assert [(float(l), s) for l, s in res[0]["micro"]] == [(float(l), s) for l, s in res[1]["micro"]]
    assert torch.equal(res[0]["grad"], res[1]["grad"]) and torch.equal(res[0]["params"], res[1]["params"])


@pytest.mark.parametrize("case", ["fused_p0.1", "scratch_p0.1"])
def test_rank_128_cuda_graph_replay_equals_eager(S, deterministic, monkeypatch, case):
    """One captured step replayed from a restored state: loss, gradient and parameters equal the eager step's bit for bit."""
    with monkeypatch.context() as mp:
        H = _rank_128(mp, S)
        bs = S.BenchStep(H, STEP_CASES[case])
        snap = (bs.gsync.flat_param.clone(), bs.gsync.flat.clone(), bs.model.dropout_seed.clone())
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                for kd in bs.kinds():
                    bs.body(*kd)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graphs = {}
        for kd in bs.kinds():
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                bs.body(*kd)
            graphs[kd] = g

        def restore():
            bs.gsync.flat_param.copy_(snap[0])
            bs.gsync.flat.copy_(snap[1])
            bs.model.dropout_seed.copy_(snap[2])
            for t in bs.opt._flat:
                t.zero_()
            bs.opt._step_dev.zero_()
            torch.cuda.synchronize()

        restore()
        eager = [bs.step(0), bs.step(1)]
        restore()
        replayed = [bs.step(0, graphs), bs.step(1, graphs)]
    for e, g in zip(eager, replayed):
        assert [(float(l), s) for l, s in e["micro"]] == [(float(l), s) for l, s in g["micro"]]
        for key in ("grad", "flat_grad", "clip", "params"):
            assert torch.equal(e[key], g[key]), key


@pytest.fixture
def deterministic(monkeypatch):
    """The attention backward and cuBLAS in their deterministic forms, as bench.py runs them (as in test_gpu_bench_step.py)."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev, prev_fill = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    torch.backends.cuda.matmul.allow_tf32 = True
    yield
    torch.use_deterministic_algorithms(prev)
    torch.utils.deterministic.fill_uninitialized_memory = prev_fill
    torch.backends.cuda.matmul.allow_tf32 = prev_tf32
