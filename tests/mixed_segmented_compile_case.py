"""Helper run in a SUBPROCESS by tests/test_gpu_mixed_segmented.py: the q/k/v (grouped) and o linears of a 4096-wide layer,
each serving 64 LoRA adapters at once through the row-index tensor form of `lora_linear4bit_group_mixed` /
`lora_linear4bit_mixed`, compiled with `torch.compile(fullgraph=True)` (aot_eager backend) and the token dimension marked
dynamic.  64 and 700 rows, two assignments each, must run one compiled frame with no graph break and give eager's bits.

usage: python mixed_segmented_compile_case.py      (prints one JSON line)
Not a test module (no test_ prefix)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from torch import nn  # noqa: E402

from test_gpu_mixed_adapters import BF16, _adapters, _base  # noqa: E402

H, NA = 4096, 64


class Attn(nn.Module):
    def __init__(self):
        super().__init__()
        import qlora_b200 as q

        self.bases = nn.ModuleList([_base(H, H, BF16, seed=90 + i) for i in range(4)])
        self.sets = [q.LoraAdapterSet(_adapters(H, H, NA, BF16, seed=9000 + 500 * i)) for i in range(4)]

    def forward(self, x, rows):
        import qlora_b200 as q

        qh, kh, vh = q.lora_linear4bit_group_mixed(x, list(self.bases[:3]), self.sets[:3], rows)
        return q.lora_linear4bit_mixed(qh + kh + vh, self.bases[3], self.sets[3], rows)


def main():
    from torch._dynamo.testing import CompileCounterWithBackend

    import compile_case as cc

    model = Attn()
    torch._dynamo.reset()
    torch._dynamo.utils.counters.clear()
    cnt = CompileCounterWithBackend("aot_eager")
    cm = torch.compile(model, fullgraph=True, backend=cnt)
    equal, outs = [], []
    with torch.no_grad():
        for m in (64, 700):
            x = (torch.randn(m, H, generator=torch.Generator().manual_seed(m)) * 0.5).to(BF16).cuda()
            for assign in ([(7 * t) % NA for t in range(m)], [-1 if t % 3 == 0 else 5 for t in range(m)]):
                rows = torch.tensor(assign, dtype=torch.int32, device="cuda")
                torch._dynamo.mark_dynamic(x, 0)
                torch._dynamo.mark_dynamic(rows, 0)
                eager = model(x, rows)
                comp = cm(x, rows)
                equal.append(bool(torch.equal(eager, comp)))
                outs.append(eager)
    return {"graph_breaks": cc.graph_breaks(), "frames": cnt.frame_count, "equal": equal,
            "assignments_differ": not torch.equal(outs[0], outs[1])}


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print(json.dumps(main()))
