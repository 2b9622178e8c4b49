"""fp16 compute (`bnb_4bit_compute_dtype=torch.float16`) against bf16 and against fp16 dequantize_4bit + cuBLAS, and bf16
compute over an fp16 quant state with fp16 activations (an fp16 checkpoint under `bnb_4bit_compute_dtype=torch.bfloat16`)
against today's unfused path and the bf16 twin, at the Llama-2-7B linear shapes.  Prints one JSON line with the card's name
and power limit.

  decode : 1, 8 and 16 tokens through the seven projections of a decoder layer (q, k, v, o, gate, up, down), CUDA graph over
           `--layers` distinct layers so that every weight comes from HBM; microseconds per layer:
             fused_fp16_lora   lora_linear4bit, fp16 base / adapters / x (lora_A projection + skinny kernel with U.V^T epilogue)
             fused_fp16        Linear4bit alone, fp16
             unfused_fp16      fp16 dequantize_4bit + F.linear (cuBLAS), the path fp16 compute took before
             fused_bf16        Linear4bit alone, bf16 (reference; the twin of the two arms below)
             fused_bf16_sf16   Linear4bit(compute bf16) over an fp16 state, fp16 x: input cast + fused launch with fp16 output
             unfused_bf16_sf16 the same module with autograd.USE_FUSED = False: x.to(bf16), fp16 dequantize_4bit, .to(bf16),
                               cuBLAS, .to(fp16)
  train  : M = 2048 tokens, forward and dX, single linears (q, gate, down shapes) and the grouped q/k/v and gate/up launches;
           microseconds per call (CUDA events, median of `--reps` windows):
             fused_fp16, fused_bf16, unfused_fp16 (dequantize_4bit + cuBLAS per linear)
             fused_bf16_sf16_of16    bf16 operands over fp16 states, fp16 output from the epilogue
             unfused_bf16_sf16_of16  fp16 dequantize_4bit, .to(bf16), cuBLAS, .to(fp16) per linear (dX: summed, then cast)

  python tools/fp16_perf.py [--layers 4] [--reps 7] [--r 64] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=4)
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--r", type=int, default=64)
ap.add_argument("--out", default=None)
args = ap.parse_args()

import torch  # noqa: E402

import qlora_b200 as q  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402

F = q.functional
H, I = 4096, 11008
SHAPES = [("q", H, H), ("k", H, H), ("v", H, H), ("o", H, H), ("gate", I, H), ("up", I, H), ("down", H, I)]
SCALING = 16 / args.r
M_TRAIN = 2048


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().splitlines()[0].split(", ") + [""])[:2] if r.returncode == 0 else (torch.cuda.get_device_name(), "")
    return name, power


def make_layer(seed, dtype, state_dtype=None):
    mods = []
    for j, (_, n, k) in enumerate(SHAPES):
        lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=dtype, quant_type="nf4", compress_statistics=True)
        lin.weight = q.nn.Params4bit(make_weight(n, k, seed=seed * 16 + j, dtype=state_dtype or dtype).cpu(), requires_grad=False,
                                     quant_type="nf4", compress_statistics=True)
        lin = lin.cuda()
        a = make_weight(args.r, k, seed=seed * 16 + j + 100, scale=0.02, dtype=dtype)
        b = make_weight(n, args.r, seed=seed * 16 + j + 200, scale=0.02, dtype=dtype)
        mods.append((lin, a, b))
    return mods


def median(ts):
    ts = sorted(ts)
    return ts[len(ts) // 2]


def graph_us(fn, windows=9):
    """Median of `windows` replays of a CUDA graph of fn(), microseconds."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s), torch.no_grad():
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fn()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
    return median(ts)


def events_us(fn, calls=10):
    """Median over `--reps` windows of `calls` back-to-back eager calls, microseconds per call."""
    with torch.no_grad():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3 / calls)
    return median(ts)


name, power = card()
res = {"tag": "fp16_perf", "gpu": name, "power_limit": power, "layers_in_graph": args.layers, "r": args.r}
layers = {dt: [make_layer(s, dt) for s in range(args.layers)] for dt in (torch.float16, torch.bfloat16)}
MIXED = "bf16_sf16"   # bf16 compute over fp16 states
layers[MIXED] = [make_layer(s, torch.bfloat16, torch.float16) for s in range(args.layers)]

# ---- decode
for tokens in (1, 8, 16):
    xs = {dt: {H: make_act(tokens, H, seed=1).to(dt).view(1, tokens, H), I: make_act(tokens, I, seed=2).to(dt).view(1, tokens, I)}
          for dt in (torch.float16, torch.bfloat16)}

    def run(lkey, dt, mode):
        def fn():
            q.autograd.USE_FUSED = mode != "module_unfused"   # routing is decided while the graph is captured
            try:
                for mods in layers[lkey]:
                    for lin, a, b in mods:
                        x = xs[dt][lin.in_features]
                        if mode == "lora":
                            q.lora.lora_linear4bit(x, lin, a, b, SCALING)
                        elif mode in ("base", "module_unfused"):
                            lin(x)
                        else:
                            torch.nn.functional.linear(x, F.dequantize_4bit(lin.weight.data, lin.weight.quant_state).to(dt))
            finally:
                q.autograd.USE_FUSED = True
        return fn

    for key, lkey, dt, mode in (("fused_fp16_lora", torch.float16, torch.float16, "lora"),
                                ("fused_fp16", torch.float16, torch.float16, "base"),
                                ("unfused_fp16", torch.float16, torch.float16, "unfused"),
                                ("fused_bf16", torch.bfloat16, torch.bfloat16, "base"),
                                ("fused_bf16_sf16", MIXED, torch.float16, "base"),
                                ("unfused_bf16_sf16", MIXED, torch.float16, "module_unfused")):
        res[f"decode_{tokens}tok_{key}_us_per_layer"] = round(graph_us(run(lkey, dt, mode)) / args.layers, 1)

# ---- training-size forward and dX (layer 0's weights)
for lkey, dt, tag in ((torch.float16, torch.float16, "fp16"), (torch.bfloat16, torch.bfloat16, "bf16"),
                      (MIXED, torch.bfloat16, "bf16_sf16_of16")):
    mods = layers[lkey][0]
    out_dtype = torch.float16 if lkey == MIXED else None
    x_h, x_i = make_act(M_TRAIN, H, seed=3).to(dt), make_act(M_TRAIN, I, seed=4).to(dt)
    dy_h, dy_i = make_act(M_TRAIN, H, seed=5).to(dt), make_act(M_TRAIN, I, seed=6).to(dt)
    x_of = {H: x_h, I: x_i}
    dy_of = {H: dy_h, I: dy_i}
    packs = [lin.weight.data for lin, _, _ in mods]
    qss = [lin.weight.quant_state for lin, _, _ in mods]
    cases = {"q": [0], "gate": [4], "down": [6], "qkv_x3": [0, 1, 2], "gateup_x2": [4, 5]}
    for cname, idx in cases.items():
        n, k = SHAPES[idx[0]][1], SHAPES[idx[0]][2]
        ps, ss = [packs[i] for i in idx], [qss[i] for i in idx]
        x, dys = x_of[k], [dy_of[n]] * len(idx)
        res[f"train_{cname}_fwd_fused_{tag}_us"] = round(events_us(
            lambda: F.nf4_linear_group(False, [x] * len(idx), ps, ss, out_dtype=out_dtype)), 1)
        res[f"train_{cname}_dx_fused_{tag}_us"] = round(events_us(lambda: F.nf4_linear_group(True, dys, ps, ss, out_dtype=out_dtype)), 1)
        if lkey != torch.bfloat16:
            def unf_fwd():
                for p, s in zip(ps, ss):
                    y = torch.nn.functional.linear(x, F.dequantize_4bit(p, s).to(dt))
                    if out_dtype is not None:
                        y.to(out_dtype)

            def unf_dx():
                dx = None
                for p, s, dy in zip(ps, ss, dys):
                    t = dy @ F.dequantize_4bit(p, s).to(dt)
                    dx = t if dx is None else dx + t
                if out_dtype is not None:
                    dx.to(out_dtype)

            res[f"train_{cname}_fwd_unfused_{tag}_us"] = round(events_us(unf_fwd), 1)
            res[f"train_{cname}_dx_unfused_{tag}_us"] = round(events_us(unf_dx), 1)

line = json.dumps(res)
print(line, flush=True)
if args.out:
    with open(args.out, "a") as f:
        f.write(line + "\n")
