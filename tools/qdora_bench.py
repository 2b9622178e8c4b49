#!/usr/bin/env python
"""QDoRA training-step throughput: the bench.py workload (Llama NF4+double-quant, adapters on all 7 linears, checkpointed
layers, clip 0.3, paged AdamW, one CUDA graph per step) with DoRA adapters, timed for the fused path (magnitude folded into
the NF4 dequant, DESIGN.md 6b) and for the peft-form restatement (W dequantized to HBM every forward for the norm, cuBLAS,
a second base GEMM under dropout) on the same model in one process.  Prints one JSON line.  The arms train the same
adapters one after the other, so the loss each reports differs by the optimizer steps in between.

  python tools/qdora_bench.py [--model llama2-7b] [--seq 2048] [--lora-r 64] [--lora-dropout 0.1] [--steps 5] [--warmup 3]
  python tools/qdora_bench.py --arms fused --dump-outputs DIR    # also write what the last fused step computed (bench.py's format)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama2-7b")
    ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--lora-r", type=int, default=64)
    ap.add_argument("--lora-dropout", type=float, default=0.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--arms", default="fused,peft", help="comma-separated subset of fused,peft (timed in this order)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="after the fused arm's timed steps, write its outputs")
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


def main():
    args = parse_args()
    arms = [a for a in args.arms.split(",") if a]
    assert arms and all(a in ("fused", "peft") for a in arms), args.arms
    # every kernel in its deterministic form, as in bench.py: two runs with the same arguments give the same outputs
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    import torch

    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    assert torch.cuda.is_available(), "qdora_bench.py needs a GPU"

    import bench
    import harness.llama_qlora as H
    import qlora_b200 as q
    from harness.dp import FlatGradSync
    from harness.llama_qlora import SHAPES, LlamaQLoRA, synthetic_batch
    from qlora_b200 import autograd as qauto
    from qlora_b200 import lora as qlora_mod

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    qlora_mod.ACCUMULATE_ADAPTER_GRADS_IN_PLACE = True   # persistent flat .grad buffers (harness/dp.py)
    torch.backends.cuda.matmul.allow_tf32 = True
    shape = SHAPES[args.model]
    model = LlamaQLoRA(shape, device, lora_r=args.lora_r, lora_alpha=16, lora_dropout=args.lora_dropout, seed=1234,
                       double_quant=True, grad_checkpointing=True, use_dora=True).train()
    params = model.trainable_parameters()
    opt = q.optim.PagedAdamW32bit(params, lr=2e-4, betas=(0.9, 0.999), weight_decay=0.0, capturable=True)
    gsync = FlatGradSync(params, 1, layer_of=model.trainable_parameter_layers(), n_buckets=1, overlap=True, flat_params=True)
    batches = [tuple(t.to(device) for t in synthetic_batch(shape, args.seq, seed=j)) for j in range(4)]
    static_ids, static_labels = batches[0][0].clone(), batches[0][1].clone()
    static_loss = torch.zeros((), device=device, dtype=torch.float32)
    clip_coef = torch.ones((), device=device, dtype=torch.float32)

    def step_body():
        gsync.zero()
        model.dropout_seed.add_(1)
        loss = model(static_ids, static_labels)
        loss.backward()
        static_loss.copy_(loss.detach())
        gsync.finish()
        torch.clamp(0.3 / (torch.linalg.vector_norm(gsync.flat, dtype=torch.float32) + 1e-6), max=1.0, out=clip_coef)
        opt.step_flat(gsync.flat_param, gsync.flat, grad_scale=clip_coef)

    def set_arm(fused: bool):
        qauto.USE_FUSED = fused
        H.GROUP_LINEARS = fused
        for mod in model.modules():
            if hasattr(mod, "fused"):
                mod.fused = fused

    results = {}
    clocks = {}
    for arm in arms:
        set_arm(arm == "fused")
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
        clocks[arm] = sampler.stop()
        secs = e0.elapsed_time(e1) / 1e3
        results[arm] = {"value": args.seq * args.steps / secs, "ms_per_step": 1e3 * secs / args.steps, "loss": static_loss.item()}
        if arm == "fused" and args.dump_outputs:
            bench.dump_outputs(args.dump_outputs, static_loss, gsync, params)
        del graph
    set_arm(True)

    line = {"metric": f"train_tokens_per_sec_{args.model.replace('-', '_')}_nf4_dq_dora_seq{args.seq}", "unit": "tokens/s",
            "fused": results.get("fused"), "peft_form": results.get("peft"), "steps": args.steps, "warmup": args.warmup,
            "workload": f"{args.model} NF4+double-quant, DoRA r={args.lora_r} alpha=16 dropout={args.lora_dropout} on all 7 linears, "
                        f"seq {args.seq}, bs 1, grad-checkpointing, paged AdamW on adapters and magnitudes, clip 0.3, one CUDA graph per step",
            "gpu": torch.cuda.get_device_name(device), "power_limit_w": power_limit(), "clocks": clocks}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
