"""Eager against torch.compile for an HF-built Llama-2-7B QLoRA training step, and the graph breaks Dynamo meets.

The model is built the reference's way: `LlamaForCausalLM` on the meta device -> `replace_with_bnb_linear`
(BitsAndBytesConfig nf4, double quant, bf16 compute) -> every Linear4bit given random bf16 weights quantized on the GPU
(`Params4bit(value, **old.__dict__).to("cuda")`).  LoRA r = 64, alpha 16, no dropout, on all seven linears of every layer,
through the library's fused `lora_linear4bit`; non-reentrant gradient checkpointing; one sequence of `--seq` tokens.

    PYTHONPATH=<repo>/shims python tools/compile_perf.py [--layers 32] [--seq 2048] [--steps 5] [--warmup 2]
    PYTHONPATH=<other tree>/shims python tools/compile_perf.py --breaks-only     # count another build's graph breaks

Prints one JSON line: the card's name and power limit, the graph breaks of `torch.compile(model, backend="eager")` over
one step, and (unless --breaks-only) eager and compiled (Inductor, default mode) milliseconds per step with the time the
first compiled step took.  Needs a GPU: there is nothing to measure without one.
"""
import argparse
import json
import math
import subprocess
import time

import torch
from torch import nn


class LoraAdapter(nn.Module):
    def __init__(self, base, r, alpha):
        super().__init__()
        self.base_layer = base
        self.lora_A = nn.Parameter(torch.empty(r, base.in_features, dtype=torch.bfloat16, device="cuda"))
        nn.init.kaiming_uniform_(self.lora_A, a=math.sqrt(5))
        self.lora_B = nn.Parameter(torch.randn(base.out_features, r, dtype=torch.bfloat16, device="cuda") * 1e-3)
        self.scaling = alpha / r

    def forward(self, x):
        import bitsandbytes as bnb

        return bnb.lora_linear4bit(x, self.base_layer, self.lora_A, self.lora_B, self.scaling)


def build(layers: int, r: int):
    import bitsandbytes as bnb
    from transformers import BitsAndBytesConfig, LlamaConfig, LlamaForCausalLM
    from transformers.integrations.bitsandbytes import replace_with_bnb_linear
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    cfg = LlamaConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=layers, num_attention_heads=32,
                      num_key_value_heads=32, vocab_size=32000, max_position_embeddings=4096, attn_implementation="sdpa")
    qcfg = BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_use_double_quant=True,
                              bnb_4bit_compute_dtype=torch.bfloat16)
    with torch.device("meta"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    model = replace_with_bnb_linear(model, modules_to_not_convert=["lm_head"], quantization_config=qcfg)
    g = torch.Generator(device="cuda").manual_seed(0)
    lin_names = [n for n, m in model.named_modules() if isinstance(m, bnb.nn.Linear4bit)]
    for n in lin_names:
        mod = model.get_submodule(n)
        value = torch.randn(mod.out_features, mod.in_features, device="cuda", generator=g, dtype=torch.bfloat16) * 0.02
        mod.weight = bnb.nn.Params4bit(value, requires_grad=False, **mod.weight.__dict__).to("cuda")
    for n, prm in list(model.named_parameters()):
        if prm.device.type == "meta":
            mod_name, _, leaf = n.rpartition(".")
            value = (torch.ones if "norm" in leaf or "norm" in mod_name else torch.randn)(
                prm.shape, device="cuda", dtype=torch.bfloat16)
            setattr(model.get_submodule(mod_name), leaf, nn.Parameter(value if "norm" in n else value * 0.02,
                                                                      requires_grad=False))
    model.model.rotary_emb = LlamaRotaryEmbedding(cfg, device="cuda")
    for n in lin_names:
        parent, _, leaf = n.rpartition(".")
        setattr(model.get_submodule(parent), leaf, LoraAdapter(model.get_submodule(n), r, 16))
    model.train()
    model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    model.disable_input_require_grads()   # its requires_grad_() hook cannot be traced; not needed when non-reentrant
    return model


def step(model, ids):
    loss = model(input_ids=ids, labels=ids, use_cache=False).loss
    loss.backward()
    for p in model.parameters():
        p.grad = None
    return loss


def time_steps(model, ids, warmup, steps):
    for _ in range(warmup):
        step(model, ids)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        step(model, ids)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def graph_breaks(model, ids):
    """Graph breaks of one step under torch.compile(backend="eager"), or the error that stopped it."""
    from torch._dynamo.utils import counters

    torch._dynamo.reset()
    counters.clear()
    try:
        step(torch.compile(model, backend="eager"), ids)
    except Exception as e:   # reported, not hidden: a build whose graph does not even break cleanly
        return {"error": f"{type(e).__name__}: {str(e).splitlines()[0][:300]}"}
    torch._dynamo.reset()
    return {"graph_breaks": sum(counters["graph_break"].values()),
            "reasons": dict(sorted(((k[:160], v) for k, v in counters["graph_break"].items()), key=lambda kv: -kv[1])[:5])}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--rank", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--breaks-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compile_perf.py needs a GPU")
    import bitsandbytes as bnb

    torch.manual_seed(0)
    model = build(args.layers, args.rank)
    ids = torch.randint(0, 32000, (1, args.seq), device="cuda")
    res = {"card": card(), "bnb_file": bnb.__file__, "layers": args.layers, "seq": args.seq, "rank": args.rank}
    res.update(graph_breaks(model, ids))
    if not args.breaks_only:
        res["eager_ms_per_step"] = time_steps(model, ids, args.warmup, args.steps)
        torch._dynamo.reset()
        cm = torch.compile(model)
        torch.cuda.synchronize()
        t = time.perf_counter()
        step(cm, ids)
        torch.cuda.synchronize()
        res["first_compiled_step_s"] = time.perf_counter() - t
        res["compiled_ms_per_step"] = time_steps(cm, ids, args.warmup, args.steps)
        res["eager_ms_per_step_after"] = time_steps(model, ids, 1, args.steps)   # eager again, for the run-to-run drift
        res["tokens_per_s"] = {"eager": args.seq * 1e3 / res["eager_ms_per_step"],
                               "compiled": args.seq * 1e3 / res["compiled_ms_per_step"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
