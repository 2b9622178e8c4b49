"""Training K DoRA (QDoRA) adapters over one NF4 base: one multi-adapter step of K*S rows against K sequential steps of S
rows and against peft's form, on the seven linears of one Llama-2-7B decoder layer, forward and backward.

Arms (each is one layer's forward + backward; the base weights are shared, every adapter has rank r on every linear):
  multi   `dora_linear4bit_group_multi` over K*S rows (q/k/v and gate/up grouped, o and down single): one step for all jobs.
  seq     K calls of `dora_linear4bit_group` on S rows each, one per adapter: what K separate jobs run.
  peft    peft's `DoraLinearLayer` restated under autograd, per adapter on its own rows (`dora_linear4bit_peft`: the base
          `Linear4bit`, a dequantized W for the norm, lora_A, lora_B and the magnitude scale).
The arms alternate within each repeat after a warmup of every arm; the time is the median over repeats of CUDA events around
the step.  Kernels per layer: CUDA kernels of one step under torch.profiler, in a pass of its own.

    python tools/multi_dora_train_perf.py [--repeats 7] [--warmup 2] [--quick]

Prints one JSON line: the GPU, its power limit, and per configuration the microseconds and kernels per layer of each arm.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D, F_ = 4096, 11008
LINEARS = {"qkv": (D, D, 3), "o": (D, D, 1), "gate_up": (F_, D, 2), "down": (D, F_, 1)}


def _query(field: str) -> str:
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _base(q, n, k, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(n, k, generator=g) * 0.02).to(torch.bfloat16)
    lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
    lin.weight = q.nn.Params4bit(w, requires_grad=False, compress_statistics=True, quant_type="nf4", module=lin)
    return lin.cuda()


class Layer:
    def __init__(self, q, n_adapters, r):
        self.q = q
        self.bases, self.ads, self.sets = {}, {}, {}
        seed = 1
        for name, (n, k, cnt) in LINEARS.items():
            self.bases[name] = [_base(q, n, k, seed + i) for i in range(cnt)]
            seed += cnt
            ads = []
            for _ in range(cnt):
                d = {}
                for a in range(n_adapters):
                    la = (torch.randn(r, k, device="cuda") * k ** -0.5).to(torch.bfloat16).requires_grad_()
                    lb = (torch.randn(n, r, device="cuda") * 0.01).to(torch.bfloat16).requires_grad_()
                    mg = (torch.rand(n, device="cuda") * 0.2 + 0.02 * k ** 0.5).to(torch.bfloat16).requires_grad_()
                    d[f"job{a}"] = (la, lb, mg, 2.0)
                ads.append(d)
            self.ads[name] = ads
            self.sets[name] = [q.DoraAdapterSet(d) for d in ads]
            for b in self.bases[name]:   # the frozen bases' row norms, cached once as a training loop would
                q.functional.weight_row_norm2(b.weight.t(), b.weight.quant_state)

    def inputs(self, name, m, seed):
        n, k, cnt = LINEARS[name]
        g = torch.Generator(device="cuda").manual_seed(seed)
        x = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16).requires_grad_()
        dys = [torch.randn(m, n, device="cuda", generator=g).to(torch.bfloat16) for _ in range(cnt)]
        return x, dys

    def multi(self, data, rows, seq, n_adapters):
        for name in LINEARS:
            x, dys = data[name]
            ys = self.q.dora_linear4bit_group_multi(x, self.bases[name], self.sets[name], rows)
            torch.autograd.backward(ys, dys)

    def seq(self, data, rows, seq, n_adapters):
        for name in LINEARS:
            x, dys = data[name]
            for a in range(n_adapters):
                sl = slice(a * seq, (a + 1) * seq)
                ads = [d[f"job{a}"] for d in self.ads[name]]
                ys = self.q.dora_linear4bit_group(x[sl], self.bases[name], [t[0] for t in ads], [t[1] for t in ads],
                                                  [t[2] for t in ads], 2.0)
                torch.autograd.backward(ys, [d[sl] for d in dys])

    def peft(self, data, rows, seq, n_adapters):
        for name in LINEARS:
            x, dys = data[name]
            ys, gs = [], []
            for base, d, dy in zip(self.bases[name], self.ads[name], dys):
                for a in range(n_adapters):
                    sl = slice(a * seq, (a + 1) * seq)
                    la, lb, mg, s = d[f"job{a}"]
                    ys.append(self.q.dora_linear4bit_peft(x[sl], base, la, lb, mg, s))
                    gs.append(dy[sl])
            torch.autograd.backward(ys, gs)


def _clear(layer):
    for ads in layer.ads.values():
        for d in ads:
            for la, lb, mg, _ in d.values():
                la.grad = lb.grad = mg.grad = None


def _time(fn, layer, *args):
    _clear(layer)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn(*args)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3


def _kernels(fn, layer, *args):
    _clear(layer)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn(*args)
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
               and not ev.name.startswith(("Memcpy", "Memset")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true", help="r = 16, K in {1, 4}, S = 256 only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_dora_train_perf: needs a CUDA GPU")
    import qlora_b200 as q

    torch.use_deterministic_algorithms(True)
    ranks, counts, seqs = ((16,), (1, 4), (256,)) if args.quick else ((16, 64), (1, 4, 16), (256, 2048))
    results = []
    for r in ranks:
        for na in counts:
            layer = Layer(q, na, r)
            for seq in seqs:
                m = na * seq
                rows = torch.arange(na, device="cuda", dtype=torch.int32).repeat_interleave(seq)
                data = {name: layer.inputs(name, m, seed=17) for name in LINEARS}
                arms = {"multi": layer.multi, "seq": layer.seq, "peft": layer.peft}
                call = (data, rows, seq, na)
                for _ in range(args.warmup):
                    for fn in arms.values():
                        _time(fn, layer, *call)
                times = {k: [] for k in arms}
                for _ in range(args.repeats):
                    for k, fn in arms.items():
                        times[k].append(_time(fn, layer, *call))
                kernels = {k: _kernels(fn, layer, *call) for k, fn in arms.items()}
                row = {"r": r, "adapters": na, "tokens_per_adapter": seq, "rows": m}
                for k in arms:
                    row[f"{k}_us"] = round(statistics.median(times[k]), 1)
                    row[f"{k}_kernels"] = kernels[k]
                results.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
                del data
            del layer
            torch.cuda.empty_cache()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": _query("power.limit"),
                      "clocks_max_sm": _query("clocks.max.sm"), "clocks_sm_after": _query("clocks.sm"), "layer": "Llama-2-7B decoder layer, "
                      "7 NF4 linears, forward + backward", "repeats": args.repeats, "warmup": args.warmup, "results": results}))


if __name__ == "__main__":
    main()
