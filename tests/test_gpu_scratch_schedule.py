"""The scratch kernel's schedule: full rounds of 256-token units taken round-robin by the CTAs, then a tail of the last
partial round cut into token ranges (nf4_gemm_wgmma.cuh, namespace sc).  Every output element must still come from one
unit summing the same products in the same order, so the grouped q/k/v and gate/up calls at token counts whose unit count
is not a multiple of the CTA count (1536, 2048 and the ragged 2000) give bitwise the fused kernel's outputs, also with
QB200_RESERVED_SMS planning for fewer CTAs (many more rounds), and a captured CUDA graph replays them bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_helpers import make_act, make_weight

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_case(path, **env):
    env = dict(os.environ, QB200_SPLITK_MAX_T="0", **env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "scratch_schedule_case.py"), str(path)],
                       capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(path)


@pytest.fixture(scope="module")
def fused_outputs(tmp_path_factory):
    return _run_case(tmp_path_factory.mktemp("fused") / "fused.npz", QB200_SCRATCH_MIN_M=str(1 << 30))


@pytest.mark.gpu
@pytest.mark.parametrize("reserved", ["0", "100"])
def test_scratch_schedule_matches_fused_kernel_bitwise(tmp_path, fused_outputs, reserved):
    """reserved = 100 leaves 32 CTAs on an H100 SXM: gate/up forward at 2048 tokens then runs 43 rounds."""
    a = _run_case(tmp_path / "scratch.npz", QB200_SCRATCH_MIN_M="1536", QB200_RESERVED_SMS=reserved)
    b = fused_outputs
    assert sorted(a.files) == sorted(b.files) and len(a.files) == 3 * (3 + 1) + 3 * (2 + 1)
    diff = [name for name in a.files if not np.array_equal(a[name], b[name])]
    assert not diff, diff


@pytest.mark.gpu
def test_scratch_schedule_replays_under_cuda_graphs():
    """Gate/up forward and dX with LoRA at a ragged 2000 tokens (rounds and a tail): graph replay equals eager."""
    import qlora_b200.functional as F
    from qlora_b200 import _lib

    m, n, k, r = 2000, 11008, 4096, 16
    ps, qss = zip(*[F.quantize_4bit(make_weight(n, k, seed=120 + i), compress_statistics=True, quant_type="nf4") for i in range(2)])
    ps = [p.t() for p in ps]
    x = make_act(m, k, seed=1)
    us = [make_act(m, r, seed=2 + i) for i in range(2)]
    vs = [make_weight(n, r, seed=4 + i) for i in range(2)]
    dys = [make_act(m, n, seed=6 + i) for i in range(2)]
    gs = [make_act(m, r, seed=8 + i) for i in range(2)]
    as_ = [make_weight(r, k, seed=10 + i) for i in range(2)]
    assert _lib.load().qb200_nf4_linear_scratch_size(2, m, n, k, 0) == 2 * n * k * 2

    def calls():
        return F.nf4_linear_group(False, [x] * 2, ps, qss, us=us, vs=vs) + [F.nf4_linear_group(True, dys, ps, qss, us=gs, vs=as_)]

    eager = calls()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):   # warm-up: tensor maps, kernel attributes, schedules
            calls()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = calls()
    for t in static:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)
