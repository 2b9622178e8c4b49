"""Runs a fixed set of NF4 linear calls and saves every output to the .npz given as argv[1] (raw bf16 / fp32 bits).

tests/test_gpu_scratch_gemm.py runs it twice, with QB200_SCRATCH_MIN_M forcing the scratch path (bf16 weight copy +
TMA-fed GEMM) and the fused path, and split-K disabled in both, then compares the two files bit for bit."""
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
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy()


def main(path):
    out = {}
    # 1000 x 1088 with r = 24: partial last feature block (forward 104 wide, dX 64), dX contraction tail 40 of 64, and a
    # LoRA step whose second k16 MMA is half zero-fill
    for (n, k, r), nested in itertools.product(((1152, 768, 16), (1000, 1088, 24)), (True, False)):
        ps, qss = zip(*[F.quantize_4bit(make_weight(n, k, seed=50 + i), compress_statistics=nested, quant_type="nf4")
                        for i in range(3)])
        ps = [p.t() for p in ps]
        for m in (64, 256, 777, 2048):
            tag = f"{n}x{k}_{int(nested)}_{m}"
            x = make_act(m, k, seed=m)
            dys = [make_act(m, n, seed=m + 1 + i) for i in range(3)]
            us = [make_act(m, r, seed=m + 10 + i) for i in range(3)]
            vs = [make_weight(n, r, seed=m + 20 + i) for i in range(3)]
            gs = [make_act(m, r, seed=m + 30 + i) for i in range(3)]
            as_ = [make_weight(r, k, seed=m + 40 + i) for i in range(3)]
            bias = make_weight(1, n, seed=m + 60).view(-1)
            out[f"fwd_{tag}"] = bits(F.nf4_linear_fwd(x, ps[0], qss[0]))
            out[f"fwd_f32_{tag}"] = bits(F.nf4_linear_fwd(x, ps[0], qss[0], out_dtype=torch.float32))
            out[f"dx_{tag}"] = bits(F.nf4_linear_bwd_dx(dys[0], ps[0], qss[0]))
            out[f"fwd_lora_bias_{tag}"] = bits(F.nf4_linear_fwd_lora(x, ps[0], qss[0], us[0], vs[0], bias))
            out[f"dx_lora_{tag}"] = bits(F.nf4_linear_bwd_dx_lora(dys[0], ps[0], qss[0], gs[0], as_[0]))
            for i, y in enumerate(F.nf4_linear_group(False, [x] * 3, ps, qss, us=us, vs=vs)):
                out[f"group_fwd_{i}_{tag}"] = bits(y)
            out[f"group_dx_{tag}"] = bits(F.nf4_linear_group(True, dys, ps, qss, us=gs, vs=as_))
    torch.cuda.synchronize()
    np.savez(path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
