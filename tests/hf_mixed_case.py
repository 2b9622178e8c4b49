"""Helper run in a SUBPROCESS by tests/test_gpu_mixed_state.py with `PYTHONPATH=<repo>/shims` — the QLoRA recipe's
`BitsAndBytesConfig(load_in_4bit, nf4, double_quant, bnb_4bit_compute_dtype=torch.bfloat16)` over an fp16 model (a Llama-2
checkpoint's dtype, which `from_pretrained(dtype="auto")` keeps) -> HF `replace_with_bnb_linear` -> `bitsandbytes.nn.Linear4bit`
on meta -> `Params4bit(value, requires_grad=False, **old.__dict__).to(device)` (HF's Bnb4bitQuantize.convert).  The state
is fp16, the compute dtype bf16 and the activations fp16.  One Linear4bit forward / backward against the oracle's
double-rounded weight, and the whole model's loss and backward.

usage: python hf_mixed_case.py      (needs a GPU; prints one JSON line)
Not a test module (no test_ prefix)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import ctypes as ct

    import numpy as np
    import torch
    import bitsandbytes as bnb  # the shim
    from transformers import BitsAndBytesConfig, LlamaConfig, LlamaForCausalLM
    from transformers.integrations.bitsandbytes import replace_with_bnb_linear

    from fp16_helpers import np32, oracle_w32
    from gpu_helpers import assert_close_bf16
    from oracle import nf4_oracle as o

    out = {"bnb_file": bnb.__file__}
    cfg = BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_use_double_quant=True,
                             bnb_4bit_compute_dtype=torch.bfloat16)
    lc = LlamaConfig(hidden_size=256, intermediate_size=704, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=4,
                     vocab_size=512, max_position_embeddings=512)
    torch.manual_seed(0)
    model = LlamaForCausalLM(lc).to(torch.float16)
    dense = {n: p.detach().clone() for n, p in model.named_parameters()}
    model = replace_with_bnb_linear(model, modules_to_not_convert=["lm_head"], quantization_config=cfg)
    lin_names = [n for n, m in model.named_modules() if isinstance(m, bnb.nn.Linear4bit)]
    out["n_linear4bit"] = len(lin_names)
    for n in lin_names:   # HF's Bnb4bitQuantize.convert, per weight
        mod = model.get_submodule(n)
        old = mod.weight
        value = dense[n + ".weight"].to("cuda")
        mod.weight = bnb.nn.Params4bit(value, requires_grad=False, **old.__dict__).to(value.device)
    for n, p in list(model.named_parameters()):   # everything else to the GPU, as from_pretrained(device_map={'': 0})
        if p.device.type != "cuda":
            mod_name, _, leaf = n.rpartition(".")
            setattr(model.get_submodule(mod_name), leaf, torch.nn.Parameter(dense[n].cuda(), requires_grad=False))
    model = model.cuda() if any(b.device.type != "cuda" for b in model.buffers()) else model
    m0 = model.get_submodule(lin_names[0])
    qs = m0.weight.quant_state
    out["compute_dtype"] = str(m0.compute_dtype)
    out["state_dtype"] = str(qs.dtype)
    assert qs.nested and m0.weight.dtype == torch.uint8

    so = os.path.join(ROOT, "oracle", "_build", "libnf4_oracle.so")
    if not os.path.exists(so):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)
    c_oracle = ct.CDLL(so)
    # packed bytes: quantized from the SAME fp16 values as the oracle's
    st = o.quantize_4bit(dense[lin_names[0] + ".weight"].float().numpy(), offset=np.float32(qs.offset.item()))
    assert np.array_equal(st["packed"], m0.weight.data.cpu().numpy().reshape(-1)), "packed bytes differ from the oracle"
    w_ref = o.bf16_round(np.asarray(oracle_w32(c_oracle, m0.weight.data, qs), np.float32).astype(np.float16).astype(np.float32))
    x = torch.randn(1, 96, m0.in_features, device="cuda", dtype=torch.float16, requires_grad=True)
    n0 = bnb.functional.LAUNCH_COUNTER[0]
    y = m0(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    out["fused_launches"] = bnb.functional.LAUNCH_COUNTER[0] - n0   # one fused launch per direction, no dequantize
    assert y.dtype == torch.float16 and x.grad.dtype == torch.float16
    xb = o.bf16_round(np32(x).reshape(96, -1))
    gyb = o.bf16_round(np32(gy).reshape(96, -1))
    assert_close_bf16(np32(y).reshape(96, -1), o.bf16_round(xb @ w_ref.T))
    assert_close_bf16(np32(x.grad).reshape(96, -1), o.bf16_round(gyb @ w_ref))
    # the weight the unfused path reads is the same
    assert np.array_equal(np32(bnb.functional.dequantize_4bit(m0.weight.data, qs).to(torch.bfloat16)), w_ref)
    # the whole HF model: causal-LM loss + backward (into the fp16 input embeddings)
    ids = torch.randint(0, 512, (1, 64), device="cuda")
    emb = model.get_input_embeddings()
    emb.weight.requires_grad_(True)
    loss = model(input_ids=ids, labels=ids).loss
    out["hf_model_loss"] = float(loss)
    assert torch.isfinite(loss)
    loss.backward()
    out["backward_ok"] = bool(emb.weight.grad is not None and torch.isfinite(emb.weight.grad.float()).all())
    out["gpu_ok"] = True
    print(json.dumps(out))


if __name__ == "__main__":
    main()
