"""GPU diagnostics for the fused kernel: each step runs in its own process (a device trap kills the
context), dumps mismatching outputs to gpurun_out/ for offline analysis.
  python tools/gpu_diag.py all            # run every step as a subprocess with a timeout
  python tools/gpu_diag.py <step>         # run one step in-process
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "gpurun_out")
os.makedirs(OUT, exist_ok=True)

STEPS = ["quant", "fwd_1cta_plain", "fwd_small", "bwd_small", "ragged", "fwd_mid", "bwd_mid", "tail_split", "perf"]  # + "prof" (for ncu)


def _setup():
    import numpy as np
    import torch

    import qlora_b200.functional as F
    from gpu_helpers import bf16_to_f32_np, make_act, make_weight, rel_err

    return np, torch, F, bf16_to_f32_np, make_act, make_weight, rel_err


def _check_linear(tag, m, n, k, nested, do_fwd=True, do_bwd=True):
    np, torch, F, to_np, make_act, make_weight, rel_err = _setup()
    w = make_weight(n, k, seed=n * 7 + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=nested, quant_type="nf4")
    wd = F.dequantize_4bit(packed, qs).float()
    res = {"tag": tag, "m": m, "n": n, "k": k, "nested": nested}
    if do_fwd:
        x = make_act(m, k, seed=1)
        y = F.nf4_linear_fwd(x, packed, qs)
        torch.cuda.synchronize()
        ref = (x.float() @ wd.t()).to(torch.bfloat16).float()
        e = rel_err(y.float().cpu().numpy(), ref.cpu().numpy())
        res["fwd_rel_err"] = e
        if not (e <= 1e-3) and m * n <= 1 << 20:
            np.savez_compressed(os.path.join(OUT, f"diag_{tag}_fwd.npz"), y=y.float().cpu().numpy(), ref=ref.cpu().numpy())
    if do_bwd:
        dy = make_act(m, n, seed=2)
        dx = F.nf4_linear_bwd_dx(dy, packed, qs)
        torch.cuda.synchronize()
        ref = (dy.float() @ wd).to(torch.bfloat16).float()
        e = rel_err(dx.float().cpu().numpy(), ref.cpu().numpy())
        res["bwd_rel_err"] = e
        if not (e <= 1e-3) and m * k <= 1 << 20:
            np.savez_compressed(os.path.join(OUT, f"diag_{tag}_bwd.npz"), y=dx.float().cpu().numpy(), ref=ref.cpu().numpy())
    print(json.dumps(res), flush=True)


def step_quant():
    np, torch, F, to_np, make_act, make_weight, rel_err = _setup()
    from oracle import nf4_oracle as o

    w = make_weight(96, 256, seed=1)
    p, qs = F.quantize_4bit(w, compress_statistics=False, quant_type="nf4")
    pr, ar = o.quantize_blockwise_nf4(w.float().cpu().numpy())
    ok1 = bool(np.array_equal(p.cpu().numpy().reshape(-1), pr) and np.array_equal(qs.absmax.cpu().numpy(), ar))
    d = F.dequantize_4bit(p, qs)
    ok2 = bool(np.array_equal(d.float().cpu().numpy(), o.dequantize_nf4(pr, ar, w.numel()).reshape(96, 256)))
    print(json.dumps({"tag": "quant", "quantize_exact": ok1, "dequantize_exact": ok2}), flush=True)


def step_perf():
    np, torch, F, to_np, make_act, make_weight, rel_err = _setup()

    def timeit(fn, iters=20, warm=5):
        for _ in range(warm):
            fn()
        flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
        ts = []
        for _ in range(iters):
            flush.zero_()  # L2 flush between timed iterations
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts.sort()
        return ts[len(ts) // 2]

    m = 2048
    for n, k in [(4096, 4096), (11008, 4096), (4096, 11008)]:
        w = make_weight(n, k, seed=n + k)
        packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
        x = make_act(m, k, seed=3)
        dy = make_act(m, n, seed=4)
        wd = F.dequantize_4bit(packed, qs)
        t_fused = timeit(lambda: F.nf4_linear_fwd(x, packed, qs))
        t_bwd = timeit(lambda: F.nf4_linear_bwd_dx(dy, packed, qs))
        t_deq = timeit(lambda: F.dequantize_4bit(packed, qs))
        t_mm = timeit(lambda: torch.nn.functional.linear(x, wd))
        t_unf = timeit(lambda: torch.nn.functional.linear(x, F.dequantize_4bit(packed, qs)))
        t_q = timeit(lambda: F.quantize_4bit(w, compress_statistics=True, quant_type="nf4"), iters=5, warm=2)
        fl = 2.0 * m * n * k
        print(json.dumps({"tag": "perf", "n": n, "k": k, "m": m, "fused_fwd_us": t_fused, "fused_bwd_us": t_bwd,
                          "dequant_us": t_deq, "cublas_us": t_mm, "unfused_us": t_unf, "quantize_us": t_q,
                          "fused_fwd_tflops": fl / t_fused / 1e6, "fused_bwd_tflops": fl / t_bwd / 1e6,
                          "cublas_tflops": fl / t_mm / 1e6, "unfused_tflops": fl / t_unf / 1e6,
                          "dequant_GBps": (n * k * 2.5 + n * k / 64) / t_deq / 1e3}), flush=True)


def run_step(name):
    if name == "quant":
        step_quant()
    elif name == "fwd_1cta_plain":
        _check_linear(name, 256, 128, 64, False, do_bwd=False)
    elif name == "fwd_small":
        _check_linear(name, 256, 128, 256, True, do_bwd=False)
    elif name == "bwd_small":
        _check_linear(name, 256, 128, 256, True, do_fwd=False)
    elif name == "ragged":
        _check_linear(name, 300, 200, 192, True)
    elif name == "fwd_mid":
        _check_linear(name, 2048, 512, 4096, True, do_bwd=False)
    elif name == "bwd_mid":
        _check_linear(name, 2048, 512, 4096, True, do_fwd=False)
    elif name == "tail_split":  # 11008-wide: 86 feature blocks, ranges that end inside a block's token strip
        _check_linear(name, 2048, 11008, 512, True)
        _check_linear(name + "_1000tok", 1000, 640, 512, True)
    elif name == "perf":
        step_perf()
    elif name == "ablate":  # fused fwd/bwd timing only (used with QB200_DEBUG_FLAGS for performance triage)
        np, torch, F, to_np, make_act, make_weight, rel_err = _setup()
        w = make_weight(4096, 4096, seed=1)
        packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
        x = make_act(2048, 4096, seed=3)
        res = {"tag": "ablate", "flags": os.environ.get("QB200_DEBUG_FLAGS", "0"), }
        for nm, fn in (("fwd", lambda: F.nf4_linear_fwd(x, packed, qs)), ("bwd", lambda: F.nf4_linear_bwd_dx(x, packed, qs))):
            for _ in range(5):
                fn()
            ts = []
            for _ in range(20):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(); e1.record(); torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            ts.sort()
            res[nm + "_us"] = ts[len(ts) // 2]
        print(json.dumps(res), flush=True)
    elif name == "prof":  # a few launches of each kernel at the 7B attention-projection size, for ncu
        np, torch, F, to_np, make_act, make_weight, rel_err = _setup()
        w = make_weight(4096, 4096, seed=1)
        packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
        x = make_act(2048, 4096, seed=3)
        for _ in range(3):
            F.nf4_linear_fwd(x, packed, qs)
            F.nf4_linear_bwd_dx(x, packed, qs)
            F.dequantize_4bit(packed, qs)
        torch.cuda.synchronize()
    elif name == "prof_shapes":  # one forward + one dX launch per Llama-2-7B layer shape (DRAM traffic per launch via ncu)
        np, torch, F, to_np, make_act, make_weight, rel_err = _setup()
        cases = []
        for n, k in [(4096, 4096), (11008, 4096), (4096, 11008)]:
            w = make_weight(n, k, seed=n + k)
            packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
            cases.append((packed, qs, make_act(2048, k, seed=3), make_act(2048, n, seed=4)))
        flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        for packed, qs, x, dy in cases:
            flush.zero_()   # cold L2, as between layers of a 3.5 GB model
            F.nf4_linear_fwd(x, packed, qs)
            flush.zero_()
            F.nf4_linear_bwd_dx(dy, packed, qs)
        torch.cuda.synchronize()
    else:
        raise SystemExit(f"unknown step {name}")


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which == "all":
        for s in STEPS:
            t0 = time.time()
            try:
                print(f"=== step {s}")
                r = subprocess.run([sys.executable, os.path.abspath(__file__), s], timeout=240, capture_output=True, text=True)
                print(f"--- step {s}: rc={r.returncode} ({time.time() - t0:.1f}s)")
                print(r.stdout[-3000:])
                if r.returncode != 0:
                    print(r.stderr[-3000:])
            except subprocess.TimeoutExpired as e:
                print(f"--- step {s}: TIMEOUT")
                print((e.stdout or b"")[-2000:], (e.stderr or b"")[-2000:])
            sys.stdout.flush()
    else:
        run_step(which)
