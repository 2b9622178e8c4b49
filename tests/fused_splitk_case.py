"""Runs single-problem forwards (bias, and LoRA + bias) and dX launches (LoRA) at the ragged shapes and few-token counts of
tests/test_gpu_fused_edges.py, and saves every output (raw bits) and the workspace each call was planned with to the .npz
given as argv[1].

tests/test_gpu_fused_edges.py runs it with QB200_RESERVED_SMS set so that the planner sees 32 CTAs: the split-K schedule
then divides the contraction 2 to 4 ways with a shorter last split, and the test checks the saved outputs against the C
oracle.  `operands` is shared with the test so that both sides see the same weights and activations."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gpu_helpers import make_act, make_weight  # noqa: E402

# (N, K, M, LoRA rank)
CASES = [(4104, 4160, 17, 24), (4104, 4160, 100, 136), (11000, 1088, 33, 56), (11000, 1088, 100, 8), (1000, 1088, 17, 72),
         (1000, 1088, 129, 24)]


def operands(F, n, k, m, r):
    """The weight (nested state), activations, bias and LoRA operands of one case."""
    packed, qs = F.quantize_4bit(make_weight(n, k, seed=n + k), compress_statistics=True, quant_type="nf4")
    return dict(packed=packed.t(), qs=qs, x=make_act(m, k, seed=m + 1), dy=make_act(m, n, seed=m + 2),
                bias=make_weight(1, n, seed=m + 3, scale=0.5).view(-1), u=make_act(m, r, seed=m + 4),
                v=make_weight(n, r, seed=m + 5, scale=0.05), g=make_act(m, r, seed=m + 6), a=make_weight(r, k, seed=m + 7, scale=0.05))


def bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy()


def main(path):
    import qlora_b200.functional as F
    from qlora_b200 import _lib

    lib = _lib.load()
    out = {}
    for n, k, m, r in CASES:
        d = operands(F, n, k, m, r)
        key = f"{n}x{k}_{m}"
        out[f"{key}_fwd_ws"] = np.int64(lib.qb200_nf4_linear_workspace_size(m, n, k, 0))
        out[f"{key}_dx_ws"] = np.int64(lib.qb200_nf4_linear_workspace_size(m, n, k, 1))
        out[f"{key}_fwd"] = bits(F.nf4_linear_fwd(d["x"], d["packed"], d["qs"], d["bias"]))
        out[f"{key}_fwd_lora"] = bits(F.nf4_linear_fwd_lora(d["x"], d["packed"], d["qs"], d["u"], d["v"], d["bias"]))
        out[f"{key}_dx_lora"] = bits(F.nf4_linear_bwd_dx_lora(d["dy"], d["packed"], d["qs"], d["g"], d["a"]))
    torch.cuda.synchronize()
    np.savez(path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
