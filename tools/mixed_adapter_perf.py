"""Mixed-adapter batches (each sequence with its own LoRA adapter, peft's `adapter_names`) at the Llama-2-7B linear shapes,
bf16 compute.  Prints one JSON line with the card's name, power limit and median SM clock over the timed windows.

  decode : 1, 8 and 16 sequences of one token with 1, 4 or 16 distinct adapters (never more than sequences), r = 16 and 64,
           through a decoder layer's linears (q/k/v grouped, o, gate/up grouped, down), a CUDA graph over `--layers` distinct
           layers so that every weight comes from HBM; microseconds per layer, the arms' replays alternated in one session:
             fused_mixed  lora_linear4bit_group_mixed / lora_linear4bit_mixed with the row-index tensor (at most 16 rows:
                          mixed projection + skinny kernel per linear; above: the segmented path)
             peft         peft's _mixed_batch_forward restated: the base Linear4bit, then per adapter index_select, lora_A,
                          lora_B, scaling multiply and index_add
             single       lora_linear4bit_group / lora_linear4bit with ONE adapter for every row (the floor)
           plus the CUDA kernels one eager layer launches in each arm (torch.profiler).
  segmented: the same, at 32, 64, 128 and 256 sequences of one token with 1, 4, 16 and 64 adapters (decode batches of a
           serving engine, above the skinny kernels' 16 rows: the segmented path).
  prefill: 16 sequences x 256 tokens, r = 64, with 4 adapters (ranks add up to 256: the names form takes the concat branch)
           and 16 adapters (the names form: one concat launch per group of at most 256 ranks); fused_mixed is the tensor
           form (the segmented path); microseconds per layer of eager calls (CUDA events), arms alternated, plus kernels
           per layer:
             concat       the names form
             fallback     the previous release's branch above 256 ranks, restated: the rows of each adapter through
                          `lora_linear4bit` (16 adapters only)
  shrink : one `lora_segmented_add` (q/k/v grouped, 16 adapters, r = 64) at 64 to 4096 rows with U from the mixed projection
           and from the segmented shrink, the two sides of `SEGMENTED_SHRINK_MIN_WORK`.

  python tools/mixed_adapter_perf.py [--layers 4] [--reps 9] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=4)
ap.add_argument("--reps", type=int, default=9)
ap.add_argument("--out", default=None)
args = ap.parse_args()

import torch  # noqa: E402

import qlora_b200 as q  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402
from qlora_b200.mixed import prefill_branch  # noqa: E402

BF16 = torch.bfloat16
H, I = 4096, 11008
SHAPES = {"q": (H, H), "k": (H, H), "v": (H, H), "o": (H, H), "gate": (I, H), "up": (I, H), "down": (H, I)}
NA_MAX = 64


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: the card's name and power limit belong to every number")
    return (r.stdout.strip().splitlines()[0].split(", ") + [""])[:2]


class ClockSampler:
    """The SM clock (MHz) polled from nvidia-smi while the timed windows run; the median goes beside every number."""

    def __init__(self):
        self.mhz, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.wait(0.25):
            r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                               capture_output=True, text=True)
            if r.returncode == 0 and r.stdout.strip().isdigit():
                self.mhz.append(int(r.stdout.strip()))

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def median(self):
        return sorted(self.mhz)[len(self.mhz) // 2] if self.mhz else None


def make_layer(seed, r):
    """{name: (Linear4bit, [(A, B, scaling)] * NA_MAX, LoraAdapterSet)}"""
    layer = {}
    for j, (nm, (n, k)) in enumerate(SHAPES.items()):
        lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=BF16, quant_type="nf4", compress_statistics=True)
        lin.weight = q.nn.Params4bit(make_weight(n, k, seed=seed * 16 + j).cpu(), requires_grad=False, quant_type="nf4",
                                     compress_statistics=True)
        lin = lin.cuda()
        ads = [(make_weight(r, k, seed=1000 * seed + 40 * j + 2 * a, scale=k ** -0.5),
                make_weight(n, r, seed=1000 * seed + 40 * j + 2 * a + 1, scale=0.02), 16 / r) for a in range(NA_MAX)]
        layer[nm] = (lin, ads, q.LoraAdapterSet({f"a{a}": t for a, t in enumerate(ads)}))
    return layer


def peft_linear(x2d, lin, ads, groups):
    """peft `_mixed_batch_forward`: base forward, then for every adapter its rows' lora_B(lora_A(x)) * scaling added back."""
    result = lin(x2d)
    for a, idx in groups:
        la, lb, s = ads[a]
        sub = x2d.index_select(0, idx)
        out = torch.nn.functional.linear(torch.nn.functional.linear(sub, la), lb) * s
        result.index_add_(0, idx, out.to(result.dtype))
    return result


def layer_fn(arm, layer, xs, rows, groups):
    L = layer
    x, xi = xs[:2]

    def fused_mixed():
        q.lora_linear4bit_group_mixed(x, [L[n][0] for n in "qkv"], [L[n][2] for n in "qkv"], rows)
        q.lora_linear4bit_mixed(x, L["o"][0], L["o"][2], rows)
        q.lora_linear4bit_group_mixed(x, [L["gate"][0], L["up"][0]], [L["gate"][2], L["up"][2]], rows)
        q.lora_linear4bit_mixed(xi, L["down"][0], L["down"][2], rows)

    def peft():
        for n in ("q", "k", "v", "o", "gate", "up"):
            peft_linear(x, L[n][0], L[n][1], groups)
        peft_linear(xi, L["down"][0], L["down"][1], groups)

    def concat():
        names = xs[2]
        q.lora_linear4bit_group_mixed(x, [L[n][0] for n in "qkv"], [L[n][2] for n in "qkv"], names)
        q.lora_linear4bit_mixed(x, L["o"][0], L["o"][2], names)
        q.lora_linear4bit_group_mixed(x, [L["gate"][0], L["up"][0]], [L["gate"][2], L["up"][2]], names)
        q.lora_linear4bit_mixed(xi, L["down"][0], L["down"][2], names)

    def fallback():
        for n in ("q", "k", "v", "o", "gate", "up", "down"):
            inp = xi if n == "down" else x
            lin = L[n][0]
            out = torch.empty((inp.shape[0], lin.out_features), dtype=BF16, device="cuda")
            for a, idx in groups:
                la, lb, s = L[n][1][a]
                out.index_copy_(0, idx, q.lora_linear4bit(inp.index_select(0, idx), lin, la, lb, s).to(BF16))

    def single():
        for names in ("qkv", ("gate", "up")):
            bs = [L[n][0] for n in names]
            q.lora_linear4bit_group(x, bs, [L[n][1][0][0] for n in names], [L[n][1][0][1] for n in names], L[names[0]][1][0][2])
        for n, inp in (("o", x), ("down", xi)):
            la, lb, s = L[n][1][0]
            q.lora_linear4bit(inp, L[n][0], la, lb, s)

    return {"fused_mixed": fused_mixed, "peft": peft, "single": single, "concat": concat, "fallback": fallback}[arm]


ARMS = ("fused_mixed", "peft", "single")


def kernels_of(fn):
    with torch.no_grad(), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
               and "Memset" not in e.name)


def capture(fns):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s), torch.no_grad():
        for f in fns:
            f()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for f in fns:
                f()
    return g


def time_alternating(runs, reps, per):
    """runs: {arm: callable}; medians over `reps` rounds, each round one window per arm in turn; microseconds / `per`."""
    ts = {a: [] for a in runs}
    for _ in range(2):
        for f in runs.values():
            f()
    torch.cuda.synchronize()
    for _ in range(reps):
        for a, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ts[a].append(e0.elapsed_time(e1) * 1e3 / per)
    return {a: sorted(v)[len(v) // 2] for a, v in ts.items()}


def assignment(m, distinct):
    idx = [t % distinct for t in range(m)]
    return idx, [f"a{a}" for a in idx]


name, power = card()
res = {"tag": "mixed_adapter_perf", "gpu": name, "power_limit": power, "layers_in_graph": args.layers, "decode": [],
       "segmented": [], "prefill": [], "shrink": []}
clock = ClockSampler()
with clock:
    for r in (16, 64):
        layers = [make_layer(s, r) for s in range(args.layers)]
        for key, tokens, counts in (("decode", (1, 8, 16), (1, 4, 16)), ("segmented", (32, 64, 128, 256), (1, 4, 16, 64))):
            for m in tokens:
                x, xi = make_act(m, H, seed=m), make_act(m, I, seed=m + 1)
                for distinct in counts:
                    if distinct > m:
                        continue
                    idx, names = assignment(m, distinct)
                    rows = layers[0]["q"][2].indices(names)
                    groups = [(a, torch.tensor([t for t in range(m) if idx[t] == a], device="cuda")) for a in sorted(set(idx))]
                    counts_k = {arm: kernels_of(layer_fn(arm, layers[0], (x, xi), rows, groups)) for arm in ARMS}
                    graphs = {arm: capture([layer_fn(arm, L, (x, xi), rows, groups) for L in layers]) for arm in ARMS}
                    us = time_alternating({a: g.replay for a, g in graphs.items()}, args.reps, args.layers)
                    row = {"r": r, "tokens": m, "adapters": distinct, "us_per_layer": us, "kernels_per_layer": counts_k}
                    res[key].append(row)
                    print(json.dumps(row), file=sys.stderr)
                    del graphs
        del layers
        torch.cuda.empty_cache()

    r, m = 64, 16 * 256
    layer = make_layer(0, r)
    x, xi = make_act(m, H, seed=5), make_act(m, I, seed=6)
    for distinct in (4, 16):
        idx = [(t // 256) % distinct for t in range(m)]      # 16 sequences of 256 tokens, sequence j on adapter j % distinct
        names = [f"a{a}" for a in idx]
        rows = layer["q"][2].indices(names)
        groups = [(a, torch.tensor([t for t in range(m) if idx[t] == a], device="cuda")) for a in sorted(set(idx))]
        arms = ARMS + ("concat",) + (("fallback",) if distinct == 16 else ())
        fns = {arm: layer_fn(arm, layer, (x, xi, names), rows, groups) for arm in arms}
        counts_k = {arm: kernels_of(f) for arm, f in fns.items()}
        with torch.no_grad():
            us = time_alternating(fns, args.reps, 1)
        res["prefill"].append({"r": r, "tokens": m, "adapters": distinct, "names_branch": prefill_branch([layer["q"][2]], names),
                               "us_per_layer": us, "kernels_per_layer": counts_k})
        print(json.dumps(res["prefill"][-1]), file=sys.stderr)

    from qlora_b200 import _ops

    threshold = _ops.SEGMENTED_SHRINK_MIN_WORK
    sets = [layer[n][2] for n in "qkv"]
    for m in (64, 128, 256, 512, 1024, 4096):
        x = make_act(m, H, seed=m)
        rows = sets[0].indices([f"a{t % 16}" for t in range(m)])
        outs = [torch.zeros((m, H), dtype=BF16, device="cuda") for _ in sets]

        def add(min_tokens):
            def f():
                _ops.SEGMENTED_SHRINK_MIN_WORK = min_tokens
                _ops.lora_segmented_add(x, [s.table for s in sets], rows, len(sets[0]), r, outs)
            return f

        with torch.no_grad():
            us = time_alternating({"project_mixed": add(1 << 30), "shrink": add(0)}, args.reps, 1)
        _ops.SEGMENTED_SHRINK_MIN_WORK = threshold
        res["shrink"].append({"r": r, "tokens": m, "adapters": 16, "us_per_add": us, "selected": "shrink" if m * len(sets) >= threshold
                              else "project_mixed"})
        print(json.dumps(res["shrink"][-1]), file=sys.stderr)
res["median_sm_clock_mhz"] = clock.median()

line = json.dumps(res)
print(line)
if args.out:
    with open(args.out, "w") as f:
        f.write(line + "\n")
