"""The scratch path of training token counts: each NF4 weight dequantized once per call into a bf16 copy, then a TMA-fed
128 x 256 wgmma GEMM (DESIGN.md 4.1).  It must read the oracle's weights bit for bit, meet the bf16 parity bar at the model
shapes, give bitwise the outputs of the fused kernel (same products, same summation order), replay under CUDA graphs, and
refuse a missing or short scratch before any launch (the last checks need no GPU)."""
import ctypes as ct
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_helpers import assert_close_bf16, bf16_to_f32_np, make_act, make_weight, oracle_weight

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-3
MODEL_SHAPES = {"7b": (2048, 4096, 11008), "13b": (2048, 5120, 13824), "65b": (2048, 8192, 22016)}
SHAPES = [(m, n, k) for m, h, i in MODEL_SHAPES.values() for n, k in ((h, h), (i, h), (h, i))]


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    return F


def _lib():
    from qlora_b200 import _lib

    return _lib.load()


def _uses_scratch(m, n, k, nprob=1, is_bwd=False):
    return _lib().qb200_nf4_linear_scratch_size(nprob, m, n, k, int(is_bwd)) == nprob * n * k * 2


def _quant(F, n, k, seed, nested=True):
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=seed), compress_statistics=nested, quant_type="nf4")
    return packed.t(), qs


@pytest.mark.gpu
@pytest.mark.parametrize("nested", [True, False])
def test_scratch_reads_bit_exact_weights(F, c_oracle, nested):
    """Identity activations make every output one product 1.0 * w: forward must return W^T and dX W, bit for bit."""
    n, k = 2304, 2048
    assert _uses_scratch(k, n, k) and _uses_scratch(n, n, k, is_bwd=True)
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=5), compress_statistics=nested, quant_type="nf4")
    w_ref = oracle_weight(packed, qs, c_oracle)
    y = F.nf4_linear_fwd(torch.eye(k, dtype=torch.bfloat16, device="cuda"), packed, qs)
    assert np.array_equal(bf16_to_f32_np(y).view(np.uint32), np.ascontiguousarray(w_ref.T).view(np.uint32))
    dx = F.nf4_linear_bwd_dx(torch.eye(n, dtype=torch.bfloat16, device="cuda"), packed, qs)
    assert np.array_equal(bf16_to_f32_np(dx).view(np.uint32), w_ref.view(np.uint32))


def _ref(a, b, extra=None):
    r = a.float() @ b.float()
    return (r if extra is None else r + extra).to(torch.bfloat16).float().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k", SHAPES)
def test_scratch_parity_at_model_shapes(F, m, n, k):
    """Forward (with bias and with LoRA), fp32 output and dX (with LoRA) against fp32 GEMMs over dequantize_4bit's weights."""
    assert _uses_scratch(m, n, k)
    r = 64
    packed, qs = _quant(F, n, k, n + k)
    wd = F.dequantize_4bit(packed, qs).t()   # [N, K]
    x, dy = make_act(m, k, seed=1), make_act(m, n, seed=2)
    u, v, g, a = make_act(m, r, seed=3), make_weight(n, r, seed=4), make_act(m, r, seed=5), make_weight(r, k, seed=6)
    bias = make_weight(1, n, seed=7).view(-1)
    xw = x.float() @ wd.float().t()
    assert_close_bf16(bf16_to_f32_np(F.nf4_linear_fwd(x, packed, qs, bias)), (xw + bias.float()).to(torch.bfloat16).float().cpu().numpy(), TOL)
    y32 = F.nf4_linear_fwd(x, packed, qs, out_dtype=torch.float32)
    assert y32.dtype == torch.float32 and torch.equal(y32, F.nf4_linear_fwd(x, packed, qs).float())
    y_l = F.nf4_linear_fwd_lora(x, packed, qs, u, v)
    assert_close_bf16(bf16_to_f32_np(y_l), (xw + u.float() @ v.float().t()).to(torch.bfloat16).float().cpu().numpy(), TOL)
    del xw
    assert_close_bf16(bf16_to_f32_np(F.nf4_linear_bwd_dx(dy, packed, qs)), _ref(dy, wd), TOL)
    assert_close_bf16(bf16_to_f32_np(F.nf4_linear_bwd_dx_lora(dy, packed, qs, g, a)), _ref(dy, wd, g.float() @ a.float()), TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("nprob,n,k", [(3, 4096, 4096), (2, 11008, 4096), (3, 5120, 5120)])
def test_scratch_grouped_parity(F, nprob, n, k):
    """q/k/v and gate/up: side-by-side forward with LoRA, and the dX contraction sum with LoRA, in one GEMM launch each."""
    m, r = 2048, 16
    assert _uses_scratch(m, n, k, nprob)
    ps, qss = zip(*[_quant(F, n, k, 13 * i + n) for i in range(nprob)])
    wds = [F.dequantize_4bit(p, s).t() for p, s in zip(ps, qss)]
    x = make_act(m, k, seed=1)
    us = [make_act(m, r, seed=10 + i) for i in range(nprob)]
    vs = [make_weight(n, r, seed=20 + i) for i in range(nprob)]
    ys = F.nf4_linear_group(False, [x] * nprob, list(ps), list(qss), us=us, vs=vs)
    for y, wd, u, v in zip(ys, wds, us, vs):
        assert_close_bf16(bf16_to_f32_np(y), _ref(x, wd.t(), u.float() @ v.float().t()), TOL)
    dys = [make_act(m, n, seed=30 + i) for i in range(nprob)]
    gs = [make_act(m, r, seed=40 + i) for i in range(nprob)]
    as_ = [make_weight(r, k, seed=50 + i) for i in range(nprob)]
    dx = F.nf4_linear_group(True, dys, list(ps), list(qss), us=gs, vs=as_)
    acc = sum(dy.float() @ wd.float() + g.float() @ a.float() for dy, wd, g, a in zip(dys, wds, gs, as_))
    assert_close_bf16(bf16_to_f32_np(dx), acc.to(torch.bfloat16).float().cpu().numpy(), TOL)


@pytest.mark.gpu
def test_scratch_and_fused_paths_are_bitwise_equal(tmp_path):
    """The same calls with the threshold forced to each side (split-K off): every output bit equal, at 64, 256, 777 (ragged)
    and 2048 tokens, single and grouped, forward and dX, with LoRA, bias and an fp32 output, at 1152 x 768 (r = 16) and at
    the ragged 1000 x 1088 (r = 24)."""
    files = {}
    for side, min_m in (("scratch", "17"), ("fused", str(1 << 30))):
        env = dict(os.environ, QB200_SCRATCH_MIN_M=min_m, QB200_SPLITK_MAX_T="0")
        files[side] = tmp_path / f"{side}.npz"
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "scratch_path_case.py"), str(files[side])],
                           capture_output=True, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
    a, b = np.load(files["scratch"]), np.load(files["fused"])
    assert sorted(a.files) == sorted(b.files) and len(a.files) == 2 * 2 * 4 * 9
    diff = [name for name in a.files if not np.array_equal(a[name], b[name])]
    assert not diff, diff


@pytest.mark.gpu
def test_fused_entry_points_without_workspace_match_the_scratch_path(F):
    """qb200_nf4_linear_fwd takes no workspace and keeps the fused kernel at 2048 tokens: bitwise the scratch path's output."""
    from qlora_b200.functional import ptr, stream_ptr

    m, n, k = 2048, 4096, 4096
    assert _uses_scratch(m, n, k)
    packed, qs = _quant(F, n, k, 3)
    x = make_act(m, k, seed=8)
    y_scratch = F.nf4_linear_fwd(x, packed, qs)
    y = torch.empty_like(y_scratch)
    p = packed.contiguous()
    rc = _lib().qb200_nf4_linear_fwd(ptr(x), ptr(p), ptr(qs.absmax), ptr(qs.state2.code), ptr(qs.state2.absmax), ptr(qs.offset),
                                     None, None, ptr(y), m, n, k, stream_ptr(x.device))
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(y, y_scratch)


@pytest.mark.gpu
def test_scratch_path_replays_under_cuda_graphs(F):
    m, n, k, r = 2048, 4096, 4096, 64
    ps, qss = zip(*[_quant(F, n, k, 70 + i) for i in range(3)])
    x = make_act(m, k, seed=1)
    us = [make_act(m, r, seed=2 + i) for i in range(3)]
    vs = [make_weight(n, r, seed=5 + i) for i in range(3)]
    dys = [make_act(m, n, seed=8 + i) for i in range(3)]
    assert _uses_scratch(m, n, k, 3)
    eager = F.nf4_linear_group(False, [x] * 3, list(ps), list(qss), us=us, vs=vs) + [F.nf4_linear_group(True, dys, list(ps), list(qss))]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):   # warm-up: tensor maps, kernel attributes, range plans
            F.nf4_linear_group(False, [x] * 3, list(ps), list(qss), us=us, vs=vs)
            F.nf4_linear_group(True, dys, list(ps), list(qss))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = F.nf4_linear_group(False, [x] * 3, list(ps), list(qss), us=us, vs=vs) + [F.nf4_linear_group(True, dys, list(ps), list(qss))]
    for t in static:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


# ---- no GPU needed: the size query and the refusal happen before any launch ----------------------------------------------

def test_scratch_size_query():
    lib = _lib()
    assert lib.qb200_nf4_linear_scratch_size(1, 16, 4096, 4096, 0) == 0
    assert lib.qb200_nf4_linear_scratch_size(3, 1 << 20, 4096, 4096, 1) == 3 * 4096 * 4096 * 2
    assert lib.qb200_nf4_linear_scratch_size(2, 1 << 20, 11008, 4096, 0) == 2 * 11008 * 4096 * 2
    assert lib.qb200_nf4_linear_scratch_size(0, 1 << 20, 4096, 4096, 0) == 0
    assert lib.qb200_nf4_linear_scratch_size(4, 1 << 20, 4096, 4096, 0) == 0


def test_missing_or_short_scratch_is_refused():
    """A training-size call without its scratch returns QB200_EINVAL (-1) with a message; nothing is launched."""
    from qlora_b200 import _lib as L

    lib = _lib()
    lib.qb200_last_error.restype = ct.c_char_p
    buf = (ct.c_char * 4096)()
    p = ct.cast(buf, ct.c_void_p).value
    p = (p + 255) & ~255
    m, n, k = 1 << 20, 128, 128
    probs = (L.Nf4Problem * 1)()
    probs[0].inp, probs[0].packed, probs[0].absmax_f32, probs[0].out = p, p, p, p
    need = lib.qb200_nf4_linear_scratch_size(1, m, n, k, 0)
    assert need == n * k * 2
    for ws, nbytes in ((None, 0), (p, need - 1), (p + 16, need)):
        assert lib.qb200_nf4_linear_group(0, 1, ct.addressof(probs), 0, m, n, k, 2, ws, nbytes, None) == -1
        assert b"scratch" in lib.qb200_last_error()
