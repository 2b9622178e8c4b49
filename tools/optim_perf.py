#!/usr/bin/env python
"""Cost of the 32-bit optimizers on the 7B adapters.  Prints one JSON line with the card's name and power limit.

1. One flat update (`step_flat` with a device-side clip coefficient, captured in a CUDA graph as bench.py runs it) over the
   7B adapters' bf16 parameters (r = 64 on all seven linears: 159 907 840), per rule: AdamW (the reference line), Lion,
   RMSprop and AdEMAMix, with the state resident and paged (unified memory, prefetched).  Reported: us per update, the bytes
   the rule must move (bf16 p and g, fp32 state: AdamW 22 B, Lion and RMSprop 14 B, AdEMAMix 30 B per element), GB/s, and
   the rate of a device-to-device `copy_` moving the same bytes (half read, half written) in the same run.
2. The 7B training step of bench.py's loop (NF4 + double quant, LoRA r = 64 on all seven linears, checkpointing, clip 0.3,
   one CUDA graph per step) with PagedAdamW32bit, PagedLion32bit and PagedAdEMAMix32bit, in that order and AdamW again
   last, in one process: tokens/s per arm.  The arms train the same adapters one after the other.

  python tools/optim_perf.py [--n 159907840] [--iters 50] [--model llama2-7b] [--seq 2048] [--steps 10] [--warmup 3] [--no-step]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BYTES_PER_ELEM = {"adamw": 2 * (2 + 4 + 4) + 2, "lion": 2 * (2 + 4) + 2, "rmsprop": 2 * (2 + 4) + 2, "ademamix": 2 * (2 + 3 * 4) + 2}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=159_907_840, help="flat adapter elements (7B, r = 64, all seven linears)")
    ap.add_argument("--iters", type=int, default=50, help="timed flat updates per rule and placement")
    ap.add_argument("--model", default="llama2-7b")
    ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-step", action="store_true", help="only the flat updates")
    return ap.parse_args()


def power_limit():
    """The card's power limit in W (read-only query): part of every number this tool prints."""
    import subprocess

    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def progress(msg):
    print(msg, file=sys.stderr, flush=True)


def make_opt(rule, params, paged):
    import qlora_b200 as q

    if rule == "adamw":
        return q.optim.AdamW(params, lr=2e-4, betas=(0.9, 0.999), weight_decay=0.0, is_paged=paged, capturable=True)
    if rule == "lion":
        return q.optim.Lion(params, lr=2e-5, betas=(0.9, 0.99), weight_decay=0.0, is_paged=paged, capturable=True)
    if rule == "rmsprop":   # no paged form
        return q.optim.RMSprop(params, lr=1e-4, alpha=0.99, eps=1e-8, weight_decay=0.0, capturable=True)
    return q.optim.AdEMAMix(params, lr=2e-4, betas=(0.9, 0.999, 0.9999), alpha=5.0, eps=1e-8, weight_decay=0.0, is_paged=paged,
                            capturable=True)


def time_graph(graph, iters):
    import torch

    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters   # us


def capture(fn):
    import torch

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def flat_updates(n, iters, device):
    import torch

    flat_p = (torch.randn(n, device=device) * 0.02).to(torch.bfloat16)
    flat_g = (torch.randn(n, device=device) * 1e-3).to(torch.bfloat16)
    clip = torch.full((), 0.5, device=device)
    out = {}
    for rule in ("adamw", "lion", "rmsprop", "ademamix"):
        for paged in (False, True):
            if rule == "rmsprop" and paged:
                continue
            opt = make_opt(rule, [torch.nn.Parameter(flat_p)], paged)
            opt.step_flat(flat_p, flat_g, grad_scale=clip)   # allocates (and for paged state, prefetches) the state
            graph = capture(lambda: opt.step_flat(flat_p, flat_g, grad_scale=clip))
            us = time_graph(graph, iters)
            nbytes = BYTES_PER_ELEM[rule] * n
            half = nbytes // 2   # a copy_ of `half` bytes reads and writes `nbytes` in all
            src = torch.empty(half, dtype=torch.uint8, device=device)
            dst = torch.empty_like(src)
            copy_graph = capture(lambda: dst.copy_(src))
            copy_us = time_graph(copy_graph, iters)
            out[f"{rule}_{'paged' if paged else 'resident'}"] = {
                "us": round(us, 1), "bytes": nbytes, "GB_per_s": round(nbytes / us / 1e3, 1),
                "copy_GB_per_s": round(nbytes / copy_us / 1e3, 1), "of_copy": round(copy_us / us, 3)}
            progress(f"flat update {rule} {'paged' if paged else 'resident'}: {out[list(out)[-1]]}")
            assert torch.isfinite(flat_p.float()).all()
            del graph, copy_graph, opt, src, dst
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    return out


def train_steps(args, device):
    import torch

    import bench
    import harness.llama_qlora as H
    from harness.dp import FlatGradSync
    from harness.llama_qlora import SHAPES, LlamaQLoRA, synthetic_batch
    from qlora_b200 import lora as qlora_mod

    qlora_mod.ACCUMULATE_ADAPTER_GRADS_IN_PLACE = True   # persistent flat .grad buffers (harness/dp.py)
    H.GROUP_LINEARS = True
    shape = SHAPES[args.model]
    model = LlamaQLoRA(shape, device, lora_r=64, lora_alpha=16, lora_dropout=0.0, seed=1234, double_quant=True,
                       grad_checkpointing=True).train()
    params = model.trainable_parameters()
    progress(f"{args.model} model built")
    gsync = FlatGradSync(params, 1, layer_of=model.trainable_parameter_layers(), n_buckets=1, overlap=True, flat_params=True)
    batches = [tuple(t.to(device) for t in synthetic_batch(shape, args.seq, seed=j)) for j in range(4)]
    static_ids, static_labels = batches[0][0].clone(), batches[0][1].clone()
    static_loss = torch.zeros((), device=device, dtype=torch.float32)
    clip_coef = torch.ones((), device=device, dtype=torch.float32)
    results, clocks = {}, {}
    names = {"adamw": "PagedAdamW32bit", "lion": "PagedLion32bit", "ademamix": "PagedAdEMAMix32bit"}
    for i, rule in enumerate(("adamw", "lion", "ademamix", "adamw")):
        opt = make_opt(rule, params, True)

        def step_body():
            gsync.zero()
            model.dropout_seed.add_(1)
            loss = model(static_ids, static_labels)
            loss.backward()
            static_loss.copy_(loss.detach())
            gsync.finish()
            torch.clamp(0.3 / (torch.linalg.vector_norm(gsync.flat, dtype=torch.float32) + 1e-6), max=1.0, out=clip_coef)
            opt.step_flat(gsync.flat_param, gsync.flat, grad_scale=clip_coef)

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                step_body()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            step_body()

        def run(n):
            for j in range(n):
                static_ids.copy_(batches[j % len(batches)][0])
                static_labels.copy_(batches[j % len(batches)][1])
                graph.replay()

        run(max(args.warmup, 1))
        torch.cuda.synchronize()
        sampler = bench.ClockSampler(0)
        sampler.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(args.steps)
        e1.record()
        torch.cuda.synchronize()
        key = names[rule] + ("_again" if i == 3 else "")
        clocks[key] = sampler.stop()
        secs = e0.elapsed_time(e1) / 1e3
        results[key] = {"tokens_per_s": round(args.seq * args.steps / secs, 1), "ms_per_step": round(1e3 * secs / args.steps, 2),
                        "loss": static_loss.item()}
        progress(f"train step {key}: {results[key]}")
        del graph, opt
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    return results, clocks


def main():
    args = parse_args()
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    import torch

    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    assert torch.cuda.is_available(), "optim_perf.py needs a GPU"
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cuda.matmul.allow_tf32 = True
    line = {"metric": "optim32_flat_update_and_7b_step", "n": args.n, "iters": args.iters,
            "flat_update": flat_updates(args.n, args.iters, device)}
    if not args.no_step:
        line["train_step"], line["clocks"] = train_steps(args, device)
        line["train_workload"] = (f"{args.model} NF4+double-quant, LoRA r=64 alpha=16 dropout=0 on all 7 linears, seq {args.seq}, bs 1, "
                                  f"grad-checkpointing, clip 0.3, one CUDA graph per step, {args.steps} timed steps per arm")
    line.update(gpu=torch.cuda.get_device_name(device), power_limit_w=power_limit())
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
