#!/usr/bin/env python
"""Peak device memory of one eager training step of the bench workload (LlamaQLoRA, NF4 + double quant, LoRA on all 7
linears, gradient checkpointing per decoder layer), as one JSON line.

  python tools/step_memory.py [--model llama2-7b] [--seq 2048] [--lora-r 64] [--no-group]

One warm-up step runs first (allocator pools, first-use work); `torch.cuda.max_memory_allocated` is then reset and read
around one more forward + backward.  The optimizer is left out: its state is the same with or without the change measured
here, and the step's peak is reached during backward."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama2-7b")
    ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--lora-r", type=int, default=64)
    ap.add_argument("--no-group", action="store_true")
    args = ap.parse_args()

    import harness.llama_qlora as H

    H.GROUP_LINEARS = not args.no_group
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    shape = H.SHAPES[args.model]
    model = H.LlamaQLoRA(shape, dev, lora_r=args.lora_r, lora_alpha=16, seed=1234, double_quant=True, grad_checkpointing=True).train()
    ids, labels = (t.to(dev) for t in H.synthetic_batch(shape, args.seq, seed=0))

    def step():
        for p in model.trainable_parameters():
            p.grad = None
        model(ids, labels).backward()
        torch.cuda.synchronize()

    step()
    resident = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    peak = torch.cuda.max_memory_allocated()
    print(json.dumps({"model": args.model, "seq": args.seq, "grouped": not args.no_group, "gpu": torch.cuda.get_device_name(dev),
                      "resident_bytes": resident, "max_memory_allocated_bytes": peak, "step_peak_over_resident_bytes": peak - resident}))


if __name__ == "__main__":
    main()
