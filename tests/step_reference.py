"""A float64 restatement of one training micro-step of the bench harness's Llama-QLoRA model (not a test module).

Plain torch on the CPU, with autograd; nothing here imports `harness` or `qlora_b200`.  The model takes as constants the
values the GPU model holds (each base weight as the C oracle dequantizes it, the bf16 embeddings, lm_head and RoPE tables,
the fp32 norm weights) and as variables the LoRA adapters, and computes what `harness.llama_qlora.LlamaQLoRA` computes:

    RMSNorm -> q/k/v = x.W^T + s.(drop(x).A^T).B^T -> RoPE (rotate_half form) -> causal softmax attention, scale 1/sqrt(d)
    -> o projection -> residual -> RMSNorm -> SwiGLU (gate, up) -> down projection -> residual; final RMSNorm -> lm_head
    -> shifted cross-entropy, ignore_index -100.

Every difference between it and the GPU step therefore comes from the GPU step's own roundings.  The dropout masks are
those of the harness's seeded dropout kernel (`dropout_kernel` in harness/csrc/fused_ops.cu), restated in numpy below.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F

LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
_SEED_MUL = 0xD1342543DE82EF95
_M64 = (1 << 64) - 1


def _splitmix64_np(z: np.ndarray) -> np.ndarray:
    """splitmix64 on uint64 arrays (wrapping arithmetic, as the kernel's)."""
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def dropout_threshold(p: float) -> int:
    """The kernel's `thr16 = uint32(p * 65536.0f + 0.5f)`, in fp32 as the kernel computes it (p arrives as a float)."""
    return int(np.float32(p) * np.float32(65536.0) + np.float32(0.5))


def dropout_keep(n: int, p: float, seed: int, salt: int) -> np.ndarray:
    """Keep mask (bool[n]) of the seeded dropout of `n` elements at step `seed` and call site `salt`.

    key = splitmix64(seed * 0xD1342543DE82EF95 + salt); vector i of 8 elements takes r0 = splitmix64(key ^ 2i) and
    r1 = splitmix64(key ^ (2i + 1)); element j of the vector is kept iff 16-bit lane j % 4 of (r0 if j < 4 else r1),
    counted from the low bits, is >= thr16."""
    assert n % 8 == 0
    key = np.uint64(int(_splitmix64_np(np.array([(int(seed) * _SEED_MUL + int(salt)) & _M64], dtype=np.uint64))[0]))
    i2 = 2 * np.arange(n // 8, dtype=np.uint64)
    words = np.stack([_splitmix64_np(key ^ i2), _splitmix64_np(key ^ (i2 + np.uint64(1)))], axis=1)   # [n/8, 2]
    lanes = words[:, :, None] >> (np.uint64(16) * np.arange(4, dtype=np.uint64))[None, None, :] & np.uint64(0xFFFF)
    return (lanes.reshape(n) >= np.uint64(dropout_threshold(p)))


@dataclass
class RefModel:
    """Constants of the GPU model, all float64 CPU tensors: `weights[(layer, linear)]` the dequantized base weights
    [out, in]; `norms[(layer, "input" | "post")]` and `final_norm` the norm weights; `embed`, `lm_head` [vocab, hidden];
    `cos`, `sin` the RoPE tables [seq, head_dim] (sin sign-folded: cat(-sin, sin)); `salts[(layer, linear)]` the dropout
    call sites."""
    weights: dict
    norms: dict
    final_norm: torch.Tensor
    embed: torch.Tensor
    lm_head: torch.Tensor
    cos: torch.Tensor
    sin: torch.Tensor
    heads: int
    eps: float
    scaling: float
    p: float = 0.0
    salts: dict = field(default_factory=dict)

    @property
    def layers(self) -> int:
        return 1 + max(i for i, _ in self.weights)


def adapter_name(layer: int, linear: str, which: str) -> str:
    """The harness's parameter name of an adapter matrix (`which` = "A" or "B")."""
    return f"layers.{layer}.{linear}.lora_{which}.weight"


def _rmsnorm(x, w, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def _rope(x, cos, sin):
    half = x.shape[-1] // 2
    return x * cos + torch.cat((x[..., half:], x[..., :half]), dim=-1) * sin


def forward(model: RefModel, adapters: dict, ids: torch.Tensor, labels: torch.Tensor, seed: int | None) -> torch.Tensor:
    """The loss of one micro-step; `adapters` maps `adapter_name(...)` to float64 tensors; `seed` is the dropout seed the
    step runs with (the value of the model's `dropout_seed`)."""
    b, s = ids.shape
    h = model.embed.shape[1]
    d = h // model.heads
    cos, sin = model.cos[:s, None, :], model.sin[:s, None, :]

    def lin(layer, name, x):
        w = model.weights[(layer, name)]
        a, bb = adapters[adapter_name(layer, name, "A")], adapters[adapter_name(layer, name, "B")]
        xl = x
        if model.p > 0:
            keep = dropout_keep(x.numel(), model.p, seed, model.salts[(layer, name)]).reshape(x.shape)
            xl = x * torch.from_numpy(keep).to(x.dtype) / (1.0 - model.p)
        return x @ w.t() + model.scaling * ((xl @ a.t()) @ bb.t())

    x = model.embed[ids]
    causal = torch.ones(s, s, dtype=torch.bool).triu(1)
    for li in range(model.layers):
        y = _rmsnorm(x, model.norms[(li, "input")], model.eps)
        q, k, v = (lin(li, n, y).view(b, s, model.heads, d) for n in ("q_proj", "k_proj", "v_proj"))
        q, k = _rope(q, cos, sin), _rope(k, cos, sin)
        q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
        scores = (q @ k.transpose(-1, -2)) / math.sqrt(d)
        att = torch.softmax(scores.masked_fill(causal, float("-inf")), dim=-1) @ v
        x = x + lin(li, "o_proj", att.transpose(1, 2).reshape(b, s, h))
        y = _rmsnorm(x, model.norms[(li, "post")], model.eps)
        x = x + lin(li, "down_proj", F.silu(lin(li, "gate_proj", y)) * lin(li, "up_proj", y))
    logits = _rmsnorm(x, model.final_norm, model.eps) @ model.lm_head.t()
    return F.cross_entropy(logits[:, :-1].reshape(-1, logits.shape[-1]), labels[:, 1:].reshape(-1), ignore_index=-100)


def micro_step(model: RefModel, adapters: dict, ids: torch.Tensor, labels: torch.Tensor, seed: int | None):
    """(loss, {name: d loss / d adapter}) of one micro-step, in float64."""
    leaves = {n: t.detach().clone().to(torch.float64).requires_grad_(True) for n, t in adapters.items()}
    loss = forward(model, leaves, ids, labels, seed)
    loss.backward()
    return float(loss.detach()), {n: t.grad for n, t in leaves.items()}
