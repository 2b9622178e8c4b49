"""Runs grouped q/k/v and gate/up calls at the Llama-2-7B shapes (forward and dX, with LoRA) at 1536, 2000 and 2048 tokens
and saves every output to the .npz given as argv[1] (raw bf16 bits).

tests/test_gpu_scratch_schedule.py runs it on the scratch path (with and without QB200_RESERVED_SMS) and on the fused path,
and compares the files bit for bit.  At these token counts the scratch kernel's unit count is not a multiple of the CTA
count, so its full rounds are followed by a tail cut into token ranges."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import qlora_b200.functional as F  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402

TOKENS = (1536, 2000, 2048)
GROUPS = {"qkv": (3, 4096, 4096), "gate_up": (2, 11008, 4096)}


def bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy()


def main(path):
    out = {}
    r = 16
    for name, (nprob, n, k) in GROUPS.items():
        ps, qss = zip(*[F.quantize_4bit(make_weight(n, k, seed=90 + i), compress_statistics=True, quant_type="nf4")
                        for i in range(nprob)])
        ps = [p.t() for p in ps]
        vs = [make_weight(n, r, seed=100 + i) for i in range(nprob)]
        as_ = [make_weight(r, k, seed=110 + i) for i in range(nprob)]
        for m in TOKENS:
            x = make_act(m, k, seed=m)
            us = [make_act(m, r, seed=m + 10 + i) for i in range(nprob)]
            dys = [make_act(m, n, seed=m + 20 + i) for i in range(nprob)]
            gs = [make_act(m, r, seed=m + 30 + i) for i in range(nprob)]
            for i, y in enumerate(F.nf4_linear_group(False, [x] * nprob, ps, qss, us=us, vs=vs)):
                out[f"{name}_fwd_{i}_{m}"] = bits(y)
            out[f"{name}_dx_{m}"] = bits(F.nf4_linear_group(True, dys, ps, qss, us=gs, vs=as_))
    torch.cuda.synchronize()
    np.savez(path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
