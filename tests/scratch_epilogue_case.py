"""Runs grouped q/k/v and gate/up calls at the Llama-2-7B shapes (forward with LoRA and bias, forward with an fp32 output,
dX with LoRA) at token counts whose scratch units end off 256- and off 32-token boundaries, and saves every output to the
.npz given as argv[1] (raw bits).  Every call runs twice and must give the same bits both times: a TMA store box that spilled
into another unit's rows would race with that unit's own store.

tests/test_gpu_scratch_epilogue.py runs it on the scratch path (with and without QB200_RESERVED_SMS) and on the fused path
and compares the files bit for bit."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import qlora_b200.functional as F  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402

TOKENS = (1552, 1808, 2000, 3000)
GROUPS = {"qkv": (3, 4096, 4096), "gate_up": (2, 11008, 4096)}


def bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy()


def main(path):
    out = {}
    r = 16
    for name, (nprob, n, k) in GROUPS.items():
        ps, qss = zip(*[F.quantize_4bit(make_weight(n, k, seed=130 + i), compress_statistics=True, quant_type="nf4")
                        for i in range(nprob)])
        ps = [p.t() for p in ps]
        vs = [make_weight(n, r, seed=140 + i) for i in range(nprob)]
        as_ = [make_weight(r, k, seed=150 + i) for i in range(nprob)]
        biases = [make_weight(1, n, seed=160 + i).view(-1) for i in range(nprob)]
        for m in TOKENS:
            x = make_act(m, k, seed=m)
            us = [make_act(m, r, seed=m + 10 + i) for i in range(nprob)]
            dys = [make_act(m, n, seed=m + 20 + i) for i in range(nprob)]
            gs = [make_act(m, r, seed=m + 30 + i) for i in range(nprob)]
            calls = {
                "fwd": lambda: F.nf4_linear_group(False, [x] * nprob, ps, qss, biases=biases, us=us, vs=vs),
                "fwd_f32": lambda: F.nf4_linear_group(False, [x] * nprob, ps, qss, out_dtype=torch.float32),
                "dx": lambda: [F.nf4_linear_group(True, dys, ps, qss, us=gs, vs=as_)],
            }
            for kind, call in calls.items():
                first = [bits(y) for y in call()]
                again = [bits(y) for y in call()]
                for i, (a, b) in enumerate(zip(first, again)):
                    assert np.array_equal(a, b), f"{name} {kind} {i} at {m} tokens differs between two identical calls"
                    out[f"{name}_{kind}_{i}_{m}"] = a
    torch.cuda.synchronize()
    np.savez(path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
