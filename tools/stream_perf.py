"""Timing of the HBM-streaming kernels of the library (SURVEY.md 8d: K1 quantize, K4 dequantize, the few-token skinny
forward) against the measured HBM copy bandwidth.

Every case is a CUDA graph of `reps` launches that rotate over enough distinct weight copies to exceed the 50 MB L2
(no flush kernels inside the timed region; every launch reads its operands from HBM), timed with CUDA events; the
per-launch figure is graph time / reps, so it includes the back-to-back launch gap a decode loop would see.

  python tools/stream_perf.py [--lib path/to/libqlora_b200.so] [--what skinny,dequant,quant,ceiling] [--out file.jsonl]

`ceiling` (with `dequant`) adds a device-to-device copy_ and a write-only fill_ at each dequantize's byte count: the
rates the same card reaches for pure streaming.  The first line names the card and its power limit.
  python tools/stream_perf.py --ncu       # one launch of each kernel after a flush, for `ncu --set full`
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ap = argparse.ArgumentParser()
ap.add_argument("--lib", default=None)
ap.add_argument("--what", default="skinny,dequant,quant")
ap.add_argument("--out", default=None)
ap.add_argument("--ncu", action="store_true")
ap.add_argument("--tag", default="")
args = ap.parse_args()

import torch  # noqa: E402

import qlora_b200._lib as _lib  # noqa: E402

if args.lib:
    _lib.LIB_PATH = os.path.abspath(args.lib)
import qlora_b200.functional as F  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402

try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    PEAK = 3350.0   # H100 SXM data sheet (HBM3)
L2_BYTES = 50 << 20   # H100 L2
SHAPES = [(4096, 4096), (11008, 4096), (4096, 11008)]
WHAT = set(args.what.split(","))
lines = []


def emit(d):
    d["lib"] = os.path.basename(_lib.LIB_PATH)
    if args.tag:
        d["tag2"] = args.tag
    print(json.dumps(d), flush=True)
    lines.append(d)


def graph_time_us(fns, reps):
    """fns: callables rotating over distinct operands; returns µs per launch of a captured graph of `reps` launches."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for f in fns:
            f()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for i in range(reps):
                fns[i % len(fns)]()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(7):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def copies_for(nbytes):
    return max(2, -(-int(1.5 * L2_BYTES) // nbytes))


def card():
    """Name and power limit of the card the numbers are measured on."""
    import subprocess

    d = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        d["power_limit"], d["max_sm_clock"] = (v.strip() for v in q.stdout.strip().split(","))
    except Exception as e:   # no nvidia-smi: the name alone
        d["power_limit"] = f"unknown ({type(e).__name__})"
    return d


def ceilings(n, k, nm, alg):
    """Two HBM ceilings at the byte count `alg` of a dequantize: a device-to-device copy_ (alg / 2 read + alg / 2 written)
    and a write-only fill_ of alg bytes."""
    half = alg // 2
    nc = copies_for(alg)
    src = [torch.empty(half, dtype=torch.uint8, device="cuda").fill_(1) for _ in range(nc)]
    dst = [torch.empty(half, dtype=torch.uint8, device="cuda") for _ in range(nc)]
    med, best = graph_time_us([(lambda s=s, d=d: d.copy_(s)) for s, d in zip(src, dst)], reps=4 * nc)
    emit({"tag": "copy_ceiling_" + nm, "n": n, "k": k, "us": round(med, 2), "us_best": round(best, 2),
          "GBps": round(2 * half / med / 1e3, 1), "frac_hbm": round(2 * half / med / 1e3 / PEAK, 3), "copies": nc})
    del src, dst
    buf = [torch.empty(alg, dtype=torch.uint8, device="cuda") for _ in range(nc)]
    med, best = graph_time_us([(lambda b=b: b.fill_(7)) for b in buf], reps=4 * nc)
    emit({"tag": "fill_ceiling_" + nm, "n": n, "k": k, "us": round(med, 2), "us_best": round(best, 2),
          "GBps": round(alg / med / 1e3, 1), "frac_hbm": round(alg / med / 1e3 / PEAK, 3), "copies": nc})
    del buf


if not args.ncu:
    emit({"tag": "card", **card()})
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")

for n, k in SHAPES:
    w = make_weight(n, k, seed=n + k)
    packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
    packed_p, qs_p = F.quantize_4bit(w, compress_statistics=False, quant_type="nf4")
    wbytes = n * k // 2 + n * k // 64
    ncopy = copies_for(wbytes)

    if "skinny" in WHAT:
        import copy

        reps_w = [(packed.clone(), copy.deepcopy(qs)) for _ in range(ncopy)]
        for m in ((1, 8) if args.ncu else tuple(int(v) for v in os.environ.get('SP_M', '1,2,4,8,16').split(','))):
            x = make_act(m, k, seed=m)
            outs = [torch.empty(m, n, dtype=torch.bfloat16, device="cuda") for _ in range(ncopy)]
            fns = [(lambda p=p, q=q, o=o: F.nf4_linear_group(False, [x], [p], [q], outs=[o])) for (p, q), o in zip(reps_w, outs)]
            if args.ncu:
                flush.zero_()
                fns[0]()
                continue
            med, best = graph_time_us(fns, reps=4 * ncopy)
            alg = wbytes + m * k * 2 + m * n * 2
            emit({"tag": "skinny", "n": n, "k": k, "m": m, "us": round(med, 2), "us_best": round(best, 2),
                  "GBps": round(alg / med / 1e3, 1), "frac_hbm": round(alg / med / 1e3 / PEAK, 3), "copies": ncopy})
        del reps_w

    if "dequant" in WHAT and (n, k) != (4096, 11008):
        for nm, (p0, q0) in (("nested", (packed, qs)), ("plain", (packed_p, qs_p))):
            import copy

            alg = n * k * 2 + n * k // 2 + (n * k // 64) * (1 if nm == "nested" else 4)
            nc = copies_for(alg)
            ins = [(p0.clone(), copy.deepcopy(q0)) for _ in range(nc)]
            outs = [torch.empty(n, k, dtype=torch.bfloat16, device="cuda") for _ in range(nc)]
            fns = [(lambda p=p, q=q, o=o: F.dequantize_4bit(p, q, out=o)) for (p, q), o in zip(ins, outs)]
            if args.ncu:
                flush.zero_()
                fns[0]()
                continue
            med, best = graph_time_us(fns, reps=4 * nc)
            emit({"tag": "dequant_" + nm, "n": n, "k": k, "us": round(med, 2), "us_best": round(best, 2),
                  "GBps": round(alg / med / 1e3, 1), "frac_hbm": round(alg / med / 1e3 / PEAK, 3), "copies": nc})
            del ins, outs
            if "ceiling" in WHAT:
                ceilings(n, k, nm, alg)

    if "quant" in WHAT and (n, k) != (4096, 11008):
        alg = n * k * 2 + n * k // 2 + (n * k // 64) * 4
        nc = copies_for(alg)
        srcs = [w.clone() for _ in range(nc)]
        lib = _lib.load()
        pk = [torch.empty(n * k // 2, dtype=torch.uint8, device="cuda") for _ in range(nc)]
        am = [torch.empty(n * k // 64, dtype=torch.float32, device="cuda") for _ in range(nc)]

        def q1(i):
            st = torch.cuda.current_stream().cuda_stream
            rc = lib.qb200_quantize_nf4(srcs[i].data_ptr(), 2, n * k, 64, pk[i].data_ptr(), am[i].data_ptr(), st)
            assert rc == 0

        fns = [(lambda i=i: q1(i)) for i in range(nc)]
        if args.ncu:
            flush.zero_()
            fns[0]()
        else:
            med, best = graph_time_us(fns, reps=4 * nc)
            emit({"tag": "quantize_nf4_bf16", "n": n, "k": k, "us": round(med, 2), "us_best": round(best, 2),
                  "GBps": round(alg / med / 1e3, 1), "frac_hbm": round(alg / med / 1e3 / PEAK, 3), "copies": nc})
        del srcs, pk, am
    torch.cuda.synchronize()

if args.out and lines:
    with open(args.out, "a") as f:
        for d in lines:
            f.write(json.dumps(d) + "\n")
