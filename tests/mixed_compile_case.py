"""Helper run in a SUBPROCESS by tests/test_gpu_mixed_adapters.py with `PYTHONPATH=<repo>/shims`: the tiny Llama of
tests/compile_case.py, each of its seven linears per layer serving three LoRA adapters at once through
`bnb.lora_linear4bit_mixed`, whose decode forward (four sequences of one token, one adapter or "__base__" each) runs under
`torch.compile(fullgraph=True)` with the aot_eager and inductor backends, and eager.

usage: python mixed_compile_case.py      (prints one JSON line)
Not a test module (no test_ prefix)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from torch import nn  # noqa: E402

import compile_case as cc  # noqa: E402

BATCH = 4


class MixedAdapter(nn.Module):
    """Three adapters over one Linear4bit; `rows` (shared by every linear) holds each token row's adapter index."""

    def __init__(self, ad, idx: int, rows: torch.Tensor):
        super().__init__()
        import bitsandbytes as bnb

        self.base_layer = ad.base_layer
        k, n = self.base_layer.in_features, self.base_layer.out_features
        adapters = {"orig": (ad.lora_A.detach(), ad.lora_B.detach(), ad.scaling)}
        for j, r in enumerate((16, 128)):
            g = torch.Generator().manual_seed(5000 + 10 * idx + j)
            a = ((torch.rand(r, k, generator=g) * 2 - 1) * k ** -0.5).to(torch.bfloat16).cuda()
            b = ((torch.rand(n, r, generator=g) * 2 - 1) * 0.02).to(torch.bfloat16).cuda()
            adapters[f"extra{j}"] = (a, b, 2.0)
        self.adapters = bnb.LoraAdapterSet(adapters)
        self.rows = rows

    def forward(self, x):
        import bitsandbytes as bnb

        return bnb.lora_linear4bit_mixed(x, self.base_layer, self.adapters, self.rows)


def main():
    from torch._dynamo.testing import CompileCounterWithBackend

    model, _, names = cc.build(False, 0.0)
    model.eval()
    rows = torch.zeros(BATCH, dtype=torch.int32, device="cuda")
    for i, n in enumerate(names):
        parent, _, leaf = n.rpartition(".")
        setattr(model.get_submodule(parent), leaf, MixedAdapter(model.get_submodule(n), i, rows))
    sets = model.get_submodule(names[0]).adapters
    ids = torch.randint(0, cc.VOCAB, (BATCH, 1), generator=torch.Generator().manual_seed(3)).cuda()
    res = {}
    # aot_eager runs the traced graph op by op: the same kernels as eager, so the same bits.  Inductor generates its own
    # kernels for the model's norms, rotary embedding and attention glue, which round differently from eager's.
    for backend in ("aot_eager", "inductor"):
        torch._dynamo.reset()
        torch._dynamo.utils.counters.clear()
        cnt = CompileCounterWithBackend(backend)
        cm = torch.compile(model, fullgraph=True, backend=cnt)
        equal, rel, outs = [], [], []
        with torch.no_grad():
            for assign in (["orig", "__base__", "extra1", "extra0"], ["extra1", "extra1", "__base__", "orig"]):
                sets.indices(assign, out=rows)
                eager = model(input_ids=ids, use_cache=False).logits
                comp = cm(input_ids=ids, use_cache=False).logits
                equal.append(bool(torch.equal(eager, comp)))
                rel.append(cc.rel(comp.double(), eager.double()))
                outs.append(eager)
        res[backend] = {"graph_breaks": cc.graph_breaks(), "frames": cnt.frame_count, "equal": equal, "rel_vs_eager": rel,
                        "assignments_differ": not torch.equal(outs[0], outs[1])}
    return res


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print(json.dumps(main()))
