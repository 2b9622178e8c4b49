"""Helper run in a SUBPROCESS by tests/test_gpu_compile.py with `PYTHONPATH=<repo>/shims`: a tiny Llama built the reference's
way (`BitsAndBytesConfig` -> HF `replace_with_bnb_linear` -> `Params4bit(value, **old.__dict__).to("cuda")`, as
tests/hf_path_case.py does), its seven linears per layer wrapped with the library's fused LoRA or DoRA, run under
`torch.compile(fullgraph=True)` and checked against a float64 restatement of the same model (the C oracle's weights).

usage: python compile_case.py <case>     (prints one JSON line)
Not a test module (no test_ prefix)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from torch import nn  # noqa: E402

HIDDEN, INTER, LAYERS, HEADS, VOCAB = 256, 704, 2, 4, 512
RANK, ALPHA, P_DROP = 64, 16, 0.1


class Adapter(nn.Module):
    """LoRA (or DoRA) over one Linear4bit through the library's fused autograd functions.  Dropout is a fixed seeded mask
    (a buffer), so a checkpoint recompute, the eager run, the compiled run and the float64 restatement all drop the same
    elements."""

    def __init__(self, base, idx: int, dora: bool, p: float, max_tokens: int):
        super().__init__()
        g = torch.Generator().manual_seed(1000 + idx)
        self.base_layer = base
        k, n = base.in_features, base.out_features
        self.lora_A = nn.Parameter((torch.rand(RANK, k, generator=g) * 2 - 1).mul(k ** -0.5).to(torch.bfloat16).cuda())
        self.lora_B = nn.Parameter((torch.rand(n, RANK, generator=g) * 2 - 1).mul(0.02).to(torch.bfloat16).cuda())
        self.scaling = ALPHA / RANK
        self.dora = dora
        if dora:
            import bitsandbytes as bnb

            norm = bnb.functional.weight_row_norm2(base.weight.data, base.weight.quant_state).sqrt()
            self.magnitude = nn.Parameter((norm * (1 + 0.1 * torch.rand(n, generator=g).cuda())).to(torch.bfloat16))
        self.p = p
        if p > 0:
            keep = (torch.rand(max_tokens, k, generator=g) >= p).to(torch.bfloat16) / (1 - p)
            self.register_buffer("mask", keep.cuda(), persistent=False)

    def lora_input(self, x):
        if self.p <= 0:
            return None
        return x * self.mask[: x.shape[-2]]

    def forward(self, x):
        import bitsandbytes as bnb

        if self.dora:
            return bnb.dora_linear4bit(x, self.base_layer, self.lora_A, self.lora_B, self.magnitude, self.scaling, self.lora_input(x))
        return bnb.lora_linear4bit(x, self.base_layer, self.lora_A, self.lora_B, self.scaling, self.lora_input(x))


class RefAdapter(nn.Module):
    """The float64 restatement of `Adapter`: peft's LoRA / DoRA forms on the oracle's weights."""

    def __init__(self, w, ad: Adapter):
        super().__init__()
        d = torch.float64
        self.w = w.to(d)
        self.lora_A = nn.Parameter(ad.lora_A.detach().to(d))
        self.lora_B = nn.Parameter(ad.lora_B.detach().to(d))
        self.magnitude = nn.Parameter(ad.magnitude.detach().to(d)) if ad.dora else None
        self.mask = ad.mask.to(d) if ad.p > 0 else None
        self.scaling = ad.scaling

    def forward(self, x):
        xl = x if self.mask is None else x * self.mask[: x.shape[-2]]
        lora = (xl @ self.lora_A.t()) @ self.lora_B.t() * self.scaling
        if self.magnitude is None:
            return x @ self.w.t() + lora
        norm = torch.linalg.norm(self.w + self.scaling * (self.lora_B @ self.lora_A), dim=1).detach()
        c = self.magnitude / norm
        if self.mask is None:
            return c * (x @ self.w.t() + lora)
        return x @ self.w.t() + (c - 1) * (xl @ self.w.t()) + c * lora


def _oracle():
    import ctypes as ct
    import subprocess

    so = os.path.join(ROOT, "oracle", "_build", "libnf4_oracle.so")
    if not os.path.exists(so):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)
    return ct.CDLL(so)


def build(dora: bool, p: float, max_tokens: int = 256):
    """(model with adapters on the GPU, float64 restatement, adapter names)."""
    import bitsandbytes as bnb
    from transformers import BitsAndBytesConfig, LlamaConfig, LlamaForCausalLM
    from transformers.integrations.bitsandbytes import replace_with_bnb_linear

    from gpu_helpers import oracle_weight

    c_oracle = _oracle()
    cfg = BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_use_double_quant=True,
                             bnb_4bit_compute_dtype=torch.bfloat16)
    lc = LlamaConfig(hidden_size=HIDDEN, intermediate_size=INTER, num_hidden_layers=LAYERS, num_attention_heads=HEADS,
                     num_key_value_heads=HEADS, vocab_size=VOCAB, max_position_embeddings=512, attn_implementation="sdpa")
    torch.manual_seed(0)
    model = LlamaForCausalLM(lc).to(torch.bfloat16)
    ref = LlamaForCausalLM(lc).to(torch.float64)
    dense = {n: p.detach().clone() for n, p in model.named_parameters()}
    model = replace_with_bnb_linear(model, modules_to_not_convert=["lm_head"], quantization_config=cfg)
    lin_names = [n for n, m in model.named_modules() if isinstance(m, bnb.nn.Linear4bit)]
    for n in lin_names:   # HF's Bnb4bitQuantize.convert, per weight
        mod = model.get_submodule(n)
        value = dense[n + ".weight"].cuda()
        mod.weight = bnb.nn.Params4bit(value, requires_grad=False, **mod.weight.__dict__).to(value.device)
    for n, prm in list(model.named_parameters()):
        if prm.device.type != "cuda":
            mod_name, _, leaf = n.rpartition(".")
            setattr(model.get_submodule(mod_name), leaf, nn.Parameter(dense[n].cuda(), requires_grad=False))
    model = model.cuda() if any(b.device.type != "cuda" for b in model.buffers()) else model
    ref.load_state_dict({k: v.to(torch.float64) for k, v in dense.items()}, strict=False)
    ref = ref.cuda()
    for prm in ref.parameters():
        prm.requires_grad_(False)
    for i, n in enumerate(lin_names):
        parent, _, leaf = n.rpartition(".")
        base = model.get_submodule(n)
        ad = Adapter(base, i, dora, p, max_tokens)
        setattr(model.get_submodule(parent), leaf, ad)
        w = torch.from_numpy(oracle_weight(base.weight.data, base.weight.quant_state, c_oracle)).cuda()
        setattr(ref.get_submodule(parent), leaf, RefAdapter(w, ad))
    return model, ref, lin_names


def adapter_grads(model, names):
    out = {}
    for n in names:
        ad = model.get_submodule(n)
        for k in ("lora_A", "lora_B", "magnitude"):
            prm = getattr(ad, k, None)
            if isinstance(prm, nn.Parameter):
                out[f"{n}.{k}"] = prm.grad.detach().double().clone()
                prm.grad = None
    return out


def step(model, ids):
    loss = model(input_ids=ids, labels=ids, use_cache=False).loss
    loss.backward()
    return loss.detach().double()


def rel(a, b):
    return float(torch.linalg.norm(a - b) / torch.linalg.norm(b).clamp_min(1e-30))


def errors(loss, grads, ref_loss, ref_grads):
    return {"loss": abs(float(loss) - float(ref_loss)) / abs(float(ref_loss)),
            "grads": {k: rel(grads[k], ref_grads[k]) for k in ref_grads}}


def graph_breaks():
    from torch._dynamo.utils import counters

    return sum(counters["graph_break"].values())


def case_model(dora: bool, ckpt: bool):
    """Compiled (fullgraph, default mode) against the float64 restatement, and against eager."""
    from torch._dynamo.testing import CompileCounterWithBackend

    p = P_DROP if ckpt else 0.0
    model, ref, names = build(dora, p)
    model.train()
    ref.train()
    if ckpt:
        model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
        model.disable_input_require_grads()   # a hook calling requires_grad_(), which Dynamo cannot trace; unneeded here
    ids = torch.randint(0, VOCAB, (2, 192), generator=torch.Generator().manual_seed(7)).cuda()
    ref_loss = step(ref, ids)
    ref_grads = adapter_grads(ref, names)
    eager_loss = step(model, ids)
    eager_grads = adapter_grads(model, names)
    torch._dynamo.reset()
    torch._dynamo.utils.counters.clear()
    cnt = CompileCounterWithBackend("inductor")
    cm = torch.compile(model, fullgraph=True, backend=cnt)
    comp_loss = step(cm, ids)
    comp_grads = adapter_grads(model, names)
    return {"graph_breaks": graph_breaks(), "frames": cnt.frame_count, "n_grads": len(ref_grads),
            "eager": errors(eager_loss, eager_grads, ref_loss, ref_grads),
            "compiled": errors(comp_loss, comp_grads, ref_loss, ref_grads),
            "compiled_vs_eager_loss": abs(float(comp_loss) - float(eager_loss)) / abs(float(eager_loss))}


def case_dynamic():
    """One compilation serves two sequence lengths: the sequence dimension marked dynamic, four sequences of 192 tokens
    (768 tokens: the fused kernel) and of 400 (1600 tokens: the scratch path), each checked against the float64
    restatement.  Four sequences keep the gradients' own noise down; lengths up to 400 keep the rounding of HF's bf16
    attention, which grows with the sequence and shows in the q / k adapters' gradients, well inside the bounds."""
    from torch._dynamo.testing import CompileCounterWithBackend

    model, ref, names = build(False, 0.0)
    model.train()
    torch._dynamo.reset()
    torch._dynamo.utils.counters.clear()
    cnt = CompileCounterWithBackend("inductor")
    cm = torch.compile(model, fullgraph=True, backend=cnt)
    res = {}
    for seq in (192, 400):
        ids = torch.randint(0, VOCAB, (4, seq), generator=torch.Generator().manual_seed(seq)).cuda()
        torch._dynamo.mark_dynamic(ids, 1)
        ref_loss = step(ref, ids)
        ref_grads = adapter_grads(ref, names)
        loss = step(cm, ids)
        res[str(seq)] = errors(loss, adapter_grads(model, names), ref_loss, ref_grads)
    return {"graph_breaks": graph_breaks(), "frames": cnt.frame_count, "by_seq": res}


def case_reduce_overhead():
    """mode="reduce-overhead" (CUDA graphs) against the default mode: the same kernels, so the same bits."""
    model, _, names = build(False, 0.0)
    model.train()
    ids = torch.randint(0, VOCAB, (2, 192), generator=torch.Generator().manual_seed(7)).cuda()
    got = {}
    for mode in ("default", "reduce-overhead"):
        torch._dynamo.reset()
        cm = torch.compile(model, fullgraph=True, mode=mode)
        for _ in range(3):   # reduce-overhead records its graph on a later call; the last call replays it
            loss = step(cm, ids)
            grads = adapter_grads(model, names)
        got[mode] = (loss, grads)
    (l0, g0), (l1, g1) = got["default"], got["reduce-overhead"]
    return {"graph_breaks": graph_breaks(), "loss_equal": bool(torch.equal(l0, l1)),
            "grads_equal": all(torch.equal(g0[k], g1[k]) for k in g0), "n_grads": len(g0)}


def case_linear_only():
    """A module made of Linear4bit calls alone, compiled against eager: bit for bit, at a skinny, a fused and a scratch
    token count, forward and dX."""
    import bitsandbytes as bnb

    torch.manual_seed(0)
    layers = []
    for k, n in ((1024, 2048), (2048, 1024), (1024, 1024)):
        lin = bnb.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
        lin.weight = bnb.nn.Params4bit(torch.randn(n, k, dtype=torch.bfloat16) * 0.02, requires_grad=False,
                                       compress_statistics=True, quant_type="nf4", module=lin)
        layers.append(lin.cuda())
    model = nn.Sequential(*layers)
    torch._dynamo.reset()
    torch._dynamo.utils.counters.clear()
    cm = torch.compile(model, fullgraph=True)
    res = {}
    for m in (8, 300, 2048):
        x = torch.randn(m, 1024, dtype=torch.bfloat16, device="cuda", requires_grad=True)
        outs = []
        for f in (model, cm):
            y = f(x)
            y.backward(torch.ones_like(y))
            outs.append((y.detach(), x.grad.clone()))
            x.grad = None
        res[str(m)] = torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    return {"graph_breaks": graph_breaks(), "equal": res}


CASES = {
    "lora": lambda: case_model(False, False),
    "dora": lambda: case_model(True, False),
    "lora_ckpt": lambda: case_model(False, True),
    "dora_ckpt": lambda: case_model(True, True),
    "reduce_overhead": case_reduce_overhead,
    "dynamic": case_dynamic,
    "linear_only": case_linear_only,
}

if __name__ == "__main__":
    torch.cuda.set_device(0)
    print(json.dumps(CASES[sys.argv[1]]()))
