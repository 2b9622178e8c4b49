"""Helper run in a SUBPROCESS by tests/test_gpu_multi_dora_train.py: a gate/up pair (grouped) and a down linear of a
1024-wide block with 1088 intermediate features, each training 16 DoRA adapters at once through `dora_linear4bit_group_multi` / `dora_linear4bit_multi`,
compiled with `torch.compile(fullgraph=True)` (aot_eager backend).  Forward and backward at 64 and 700 rows, two
assignments each, must trace without a graph break and give eager's bits; a new assignment reuses the compiled frame.

usage: python multi_dora_compile_case.py      (prints one JSON line)
Not a test module (no test_ prefix)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from torch import nn  # noqa: E402

from test_gpu_multi_dora_train import BF16, _adapters, _base  # noqa: E402

H, F_, NA = 1024, 1088, 16


class Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        import qlora_b200 as q
        from qlora_b200 import functional as F

        self.up = nn.ModuleList([_base(F_, H, BF16, BF16, seed=90 + i) for i in range(2)])
        self.down = _base(H, F_, BF16, BF16, seed=95)
        self.sets = [q.DoraAdapterSet(_adapters(F_, H, NA, BF16, seed=9000 + 500 * i)) for i in range(2)]
        self.down_set = q.DoraAdapterSet(_adapters(H, F_, NA, BF16, seed=9900))
        for b in list(self.up) + [self.down]:   # the frozen bases' row norms, cached before tracing
            F.weight_row_norm2(b.weight.t(), b.weight.quant_state)

    def forward(self, x, rows):
        import qlora_b200 as q

        g, u = q.dora_linear4bit_group_multi(x, list(self.up), self.sets, rows)
        return q.dora_linear4bit_multi(torch.nn.functional.silu(g) * u, self.down, self.down_set, rows)


def main():
    from torch._dynamo.testing import CompileCounterWithBackend

    import compile_case as cc

    model = Mlp()
    params = [t for s in model.sets + [model.down_set] for t in s.lora_as + s.lora_bs + s.magnitudes]
    torch._dynamo.reset()
    torch._dynamo.utils.counters.clear()
    cnt = CompileCounterWithBackend("aot_eager")
    cm = torch.compile(model, fullgraph=True, backend=cnt)
    equal = []
    for m in (64, 700):
        x = (torch.randn(m, H, generator=torch.Generator().manual_seed(m)) * 0.5).to(BF16).cuda()
        for assign in ([(7 * t) % NA for t in range(m)], [-1 if t % 3 == 0 else 5 for t in range(m)]):
            rows = torch.tensor(assign, dtype=torch.int32, device="cuda")
            res = []
            for fn in (model, cm):
                xi = x.detach().requires_grad_()
                y = fn(xi, rows)
                grads = torch.autograd.grad(y.float().square().sum(), [xi] + params)
                res.append([y.detach()] + list(grads))
            equal.append(all(torch.equal(a, b) for a, b in zip(*res)))
    return {"graph_breaks": cc.graph_breaks(), "frames": cnt.frame_count, "equal": equal}


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print(json.dumps(main()))
