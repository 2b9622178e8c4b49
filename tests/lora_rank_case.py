"""Runs NF4 linear calls with LoRA ranks above 64 and saves every output to the .npz given as argv[1] (raw bf16 bits).

tests/test_gpu_lora_rank.py runs it twice, with QB200_SCRATCH_MIN_M forcing the scratch path and the fused path and split-K
disabled in both, then compares the two files bit for bit: both kernels add the LoRA steps of ranks 0-63, 64-127, ... after
the NF4 steps, in the same order."""
import itertools
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import qlora_b200.functional as F  # noqa: E402
from gpu_helpers import make_act, make_weight  # noqa: E402


def bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy()


def main(path):
    out = {}
    # 1000 x 1088: partial last feature block (forward 104 wide, dX 64) and a dX contraction tail of 40
    for (n, k), r, nested in itertools.product(((1000, 1088), (4096, 4096)), (128, 200, 256), (True, False)):
        ps, qss = zip(*[F.quantize_4bit(make_weight(n, k, seed=70 + i), compress_statistics=nested, quant_type="nf4")
                        for i in range(3)])
        ps = [p.t() for p in ps]
        for m in (256, 777, 2048):
            tag = f"{n}x{k}_r{r}_{int(nested)}_{m}"
            x = make_act(m, k, seed=m)
            dys = [make_act(m, n, seed=m + 1 + i) for i in range(3)]
            ubuf = make_act(m, 3 * r, seed=m + 10)   # U (and G) of q/k/v as column slices of one buffer
            us = [ubuf[:, i * r:(i + 1) * r] for i in range(3)]
            vs = [make_weight(n, r, seed=m + 20 + i, scale=0.05) for i in range(3)]
            gbuf = make_act(m, 3 * r, seed=m + 30)
            gs = [gbuf[:, i * r:(i + 1) * r] for i in range(3)]
            as_ = [make_weight(r, k, seed=m + 40 + i, scale=0.05) for i in range(3)]
            bias = make_weight(1, n, seed=m + 60).view(-1)
            out[f"fwd_lora_bias_{tag}"] = bits(F.nf4_linear_fwd_lora(x, ps[0], qss[0], us[0].contiguous(), vs[0], bias))
            out[f"dx_lora_{tag}"] = bits(F.nf4_linear_bwd_dx_lora(dys[0], ps[0], qss[0], gs[0].contiguous(), as_[0]))
            for i, y in enumerate(F.nf4_linear_group(False, [x] * 3, ps, qss, us=us, vs=vs)):
                out[f"qkv_fwd_{i}_{tag}"] = bits(y)
            for i, y in enumerate(F.nf4_linear_group(False, [x] * 2, ps[:2], qss[:2], us=us[:2], vs=vs[:2])):
                out[f"gate_up_fwd_{i}_{tag}"] = bits(y)
            out[f"qkv_dx_{tag}"] = bits(F.nf4_linear_group(True, dys, ps, qss, us=gs, vs=as_))
            out[f"gate_up_dx_{tag}"] = bits(F.nf4_linear_group(True, dys[:2], ps[:2], qss[:2], us=gs[:2], vs=as_[:2]))
    torch.cuda.synchronize()
    np.savez(path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
