"""Per-launch timings of the fused wgmma kernel at the model shapes bench.py runs (CUDA events, L2 flushed between iterations,
median of N): single, fused-LoRA and grouped launches next to cuBLAS on pre-dequantized bf16 weights and to the
bnb-equivalent dequantize + cuBLAS sequence.  One JSON line per case on stdout.

  python tools/pair_perf.py layer [7b|13b|65b]     # the launches of one decoder layer
  python tools/pair_perf.py msweep                 # 4096x4096 forward / dX for 17..4096 tokens
  python tools/pair_perf.py one M N K [bwd]        # a single shape (used for env-variable sweeps of the cost model)
Environment knobs read by the library (static per process): QB200_COST_DQ, QB200_COST_UNIT, QB200_COST_TOK_X100,
QB200_COST_DRAIN_X100, QB200_COST_SCRATCH_STEP, QB200_SPLITK_MAX_T, QB200_SCRATCH_MIN_M (17 forces the scratch path of
training token counts, a huge value the fused kernel: run msweep once each way to place the crossover), QB200_PDL,
QB200_DEBUG_FLAGS.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import qlora_b200.functional as F  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402

_flush = None


def timeit(fn, iters=15, warm=4):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        _flush.zero_()  # L2 flush between timed iterations
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def timeit_b2b(fn, reps=20, warm=4):
    """Back-to-back launches (no flush): what a graph replay sees; includes the PDL overlap between consecutive launches."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def emit(**kw):
    print(json.dumps(kw), flush=True)


def quant(n, k, seed):
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=seed), compress_statistics=True, quant_type="nf4")
    return packed.t(), qs


def case_single(m, n, k, r=64, baselines=True, tag="single"):
    p, qs = quant(n, k, n + k)
    x, dy = make_act(m, k, seed=3), make_act(m, n, seed=4)
    u = make_act(m, r, seed=5)
    v = make_weight(n, r, seed=6)
    a = make_weight(r, k, seed=7)
    fl = 2.0 * m * n * k
    res = {"tag": tag, "m": m, "n": n, "k": k}
    res["fwd_us"] = timeit(lambda: F.nf4_linear_fwd(x, p, qs))
    res["dx_us"] = timeit(lambda: F.nf4_linear_bwd_dx(dy, p, qs))
    res["fwd_lora_us"] = timeit(lambda: F.nf4_linear_fwd_lora(x, p, qs, u, v))
    res["dx_lora_us"] = timeit(lambda: F.nf4_linear_bwd_dx_lora(dy, p, qs, u, a))
    res["fwd_b2b_us"] = timeit_b2b(lambda: F.nf4_linear_fwd(x, p, qs))
    res["dx_b2b_us"] = timeit_b2b(lambda: F.nf4_linear_bwd_dx(dy, p, qs))
    res["fwd_tflops"] = fl / res["fwd_us"] / 1e6
    res["dx_tflops"] = fl / res["dx_us"] / 1e6
    if baselines:
        wd = F.dequantize_4bit(p, qs)          # [K, N] view (transposed packed)
        wd = wd.t().contiguous()
        res["cublas_fwd_us"] = timeit(lambda: torch.nn.functional.linear(x, wd))
        res["cublas_dx_us"] = timeit(lambda: dy @ wd)
        res["dequant_us"] = timeit(lambda: F.dequantize_4bit(p, qs))
        res["unfused_fwd_us"] = timeit(lambda: torch.nn.functional.linear(x, F.dequantize_4bit(p, qs).t()))
        res["unfused_dx_us"] = timeit(lambda: dy @ F.dequantize_4bit(p, qs).t())
    emit(**res)


def case_group(m, n, k, nprob, r=64):
    ps, qss = zip(*[quant(n, k, 17 * i + n + k) for i in range(nprob)])
    x = make_act(m, k, seed=3)
    dys = [make_act(m, n, seed=10 + i) for i in range(nprob)]
    u_cat = make_act(m, nprob * r, seed=5)
    us = [u_cat[:, i * r:(i + 1) * r] for i in range(nprob)]
    vs = [make_weight(n, r, seed=20 + i) for i in range(nprob)]
    gs = [make_act(m, r, seed=30 + i) for i in range(nprob)]
    as_ = [make_weight(r, k, seed=40 + i) for i in range(nprob)]
    fl = 2.0 * m * n * k * nprob
    res = {"tag": "group", "m": m, "n": n, "k": k, "nprob": nprob}
    res["fwd_lora_us"] = timeit(lambda: F.nf4_linear_group(False, [x] * nprob, list(ps), list(qss), us=us, vs=vs))
    res["dx_lora_us"] = timeit(lambda: F.nf4_linear_group(True, dys, list(ps), list(qss), us=gs, vs=as_))
    res["fwd_us"] = timeit(lambda: F.nf4_linear_group(False, [x] * nprob, list(ps), list(qss)))
    res["dx_us"] = timeit(lambda: F.nf4_linear_group(True, dys, list(ps), list(qss)))
    res["fwd_tflops"] = fl / res["fwd_us"] / 1e6
    res["dx_tflops"] = fl / res["dx_us"] / 1e6
    # the same work as separate launches, back to back
    res["separate_fwd_lora_us"] = timeit(lambda: [F.nf4_linear_fwd_lora(x, ps[i], qss[i], us[i].contiguous(), vs[i]) for i in range(nprob)])
    res["separate_dx_lora_us"] = timeit(lambda: [F.nf4_linear_bwd_dx_lora(dys[i], ps[i], qss[i], gs[i], as_[i]) for i in range(nprob)])
    emit(**res)


MODELS = {"7b": (4096, 11008, 2048), "13b": (5120, 13824, 2048), "65b": (8192, 22016, 1024)}


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "layer"
    emit(tag="env", **{k: v for k, v in os.environ.items() if k.startswith("QB200_")})
    if mode == "layer":
        h, i, m = MODELS[sys.argv[2] if len(sys.argv) > 2 else "7b"]
        case_single(m, h, h)
        case_single(m, i, h)
        case_single(m, h, i)
        case_group(m, h, h, 3)
        case_group(m, i, h, 2)
    elif mode == "msweep":
        for m in (17, 32, 64, 128, 256, 512, 1024, 2048, 4096):
            case_single(m, 4096, 4096, tag="msweep")
    elif mode == "one":
        m, n, k = (int(a) for a in sys.argv[2:5])
        case_single(m, n, k, baselines=False, tag="one")
    elif mode == "quick":   # the two launches that matter most, no baselines (cost-model sweeps)
        case_single(2048, 4096, 4096, baselines=False, tag="quick")
        case_group(2048, 4096, 4096, 3)


if __name__ == "__main__":
    main()
