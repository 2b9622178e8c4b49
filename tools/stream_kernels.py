"""Runs each streaming kernel (quantize K1, 8-bit K2/K3, dequantize K4/nested) a few times at Llama-2-7B layer sizes —
the workload for `ncu --set full -k regex:quantize|dequantize` and for the HBM-roofline numbers in profiles/."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import qlora_b200.functional as F
from qlora_b200 import _lib
from qlora_b200._lib import ptr, stream_ptr


PROF = bool(int(os.environ.get("QB200_PROF", "0")))   # under ncu: one warm-up + one timed launch per kernel


def ev_time(fn, iters=10, warm=3):
    if PROF:
        iters, warm = 1, 1
    for _ in range(warm):
        fn()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    lib = _lib.load()
    dev = torch.device("cuda")
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = peaks.get("hbm_gbs", 3350.0)   # H100 SXM data sheet (HBM3)
    only_gemv = bool(int(os.environ.get("QB200_ONLY_GEMV", "0")))
    for n, k in ((4096, 4096), (11008, 4096), (4096, 11008)):
        nel = n * k
        w = (torch.randn(n, k, device=dev) * 0.02).to(torch.bfloat16)
        packed, qs = F.quantize_4bit(w, compress_statistics=True, quant_type="nf4")
        for m in [int(v) for v in os.environ.get("QB200_GEMV_MS", "1,4,16,32").split(",")]:
            x = torch.randn(m, k, device=dev, dtype=torch.bfloat16)
            t_g = ev_time(lambda: F.nf4_linear_fwd(x, packed, qs, None))
            g_bytes = nel / 2 + nel / 64 + nel / 16384 * 4 + 1028 + 2 * m * (n + k)
            print(json.dumps({"tag": "gemv", "m": m, "n": n, "k": k, "us": t_g, "GBps": g_bytes / t_g / 1e3,
                              "frac_hbm": g_bytes / t_g / 1e3 / peak}), flush=True)
        if only_gemv:
            continue
        absmax = torch.empty(nel // 64, device=dev, dtype=torch.float32)
        out_p = torch.empty(nel // 2, device=dev, dtype=torch.uint8)
        out_w = torch.empty(n, k, device=dev, dtype=torch.bfloat16)
        s = stream_ptr(dev)
        t_q = ev_time(lambda: lib.qb200_quantize_nf4(ptr(w), 2, nel, 64, ptr(out_p), ptr(absmax), s))
        s2 = qs.state2
        t_d = ev_time(lambda: lib.qb200_dequantize_nf4_nested(ptr(packed), ptr(qs.absmax), ptr(s2.code), ptr(s2.absmax), ptr(qs.offset),
                                                               nel, 64, 256, ptr(out_w), 2, s))
        am = F.dequantize_blockwise(qs.absmax, s2) + qs.offset
        t_dp = ev_time(lambda: lib.qb200_dequantize_nf4(ptr(packed), ptr(am), nel, 64, ptr(out_w), 2, s))
        q_bytes = nel * 2 + nel / 2 + nel / 64 * 4
        d_bytes = nel / 2 + nel / 64 + nel / 16384 * 4 + 1028 + nel * 2
        print(json.dumps({"tag": "stream", "n": n, "k": k, "quantize_us": t_q, "quantize_GBps": q_bytes / t_q / 1e3,
                          "quantize_frac_hbm": q_bytes / t_q / 1e3 / peak, "dequant_nested_us": t_d,
                          "dequant_nested_GBps": d_bytes / t_d / 1e3, "dequant_nested_frac_hbm": d_bytes / t_d / 1e3 / peak,
                          "dequant_plain_us": t_dp, "hbm_peak_GBps": peak}), flush=True)


if __name__ == "__main__":
    main()
