"""The grouped forwards of tests/test_gpu_group_inputs.py, whose problems read different inputs: the cases, their operands and
the call, shared by the test and by this script.

Run as a script (argv[1]: an .npz path), it records the kernels each case's grouped call launches and each problem's output
of the single-problem call on its own operands (raw bits), for the test to compare with the grouped outputs bit for bit.
The test runs it in a subprocess of its own with QB200_SPLITK_MAX_T=0, so that no single-problem call takes the split-K
schedule, which a grouped call never takes; it profiles in that process for the reason fused_kernel_names_case.py gives."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gpu_helpers import make_act, make_weight  # noqa: E402

BF16, H16, F32 = torch.bfloat16, torch.float16, torch.float32
# (N, K, problems): q/k/v, gate/up, and two ragged shapes (a last forward feature tile 104 and 8 wide)
SHAPES = {"4096x4096": (4096, 4096, 3), "11008x4096": (11008, 4096, 2), "1000x1088": (1000, 1088, 3), "4104x4160": (4104, 4160, 2)}
# token counts by the path a grouped bf16 forward takes: the skinny kernels (1: the 1-token kernel), the fused kernel's
# range schedule (grouped calls never split K), the scratch path
TOKENS = {"skinny": (1, 5, 16), "range": (17, 300, 1535), "scratch": (1536, 1543, 2048)}
VARIANTS = ("nested", "plain", "lora16", "lora136", "bias", "row_scales", "out_f32", "out_f16", "f16_compute", "f16_state")


def _cases():
    """Every variant at one token count of each class, the counts and shapes cycling so that each appears."""
    cases = []
    shape_ids = list(SHAPES)
    for vi, variant in enumerate(VARIANTS):
        for ci, cls in enumerate(TOKENS):
            m = TOKENS[cls][vi % 3]
            cases.append((variant, m, shape_ids[(vi + ci) % len(shape_ids)]))
    return cases


CASES = _cases()


def case_id(case):
    variant, m, shape = case
    return f"{variant}-{m}-{shape}"


def dtypes(variant):
    """(compute dtype, state dtype, output dtype) of a variant."""
    cdt = H16 if variant == "f16_compute" else BF16
    sdt = H16 if variant in ("f16_compute", "f16_state") else BF16
    out = {"out_f32": F32, "out_f16": H16}.get(variant, cdt)
    return cdt, sdt, out


_WEIGHTS = {}


def weights(F, n, k, nprob, nested, sdt):
    """(packed [K/2 x N] views, quant states) of the problems' weights: the same weights for every case of a shape and state."""
    key = (n, k, nprob, nested, sdt)
    if key not in _WEIGHTS:
        ps, qss = [], []
        for i in range(nprob):
            packed, qs = F.quantize_4bit(make_weight(n, k, seed=97 * i + n + k, dtype=sdt), compress_statistics=nested,
                                         quant_type="nf4")
            ps.append(packed.t())
            qss.append(qs)
        _WEIGHTS[key] = (ps, qss)
    ps, qss = _WEIGHTS[key]
    return list(ps), list(qss)


def operands(F, case):
    """The grouped call's operands, one input (and U, V, bias, row scale) per problem, all contiguous."""
    variant, m, shape = case
    n, k, nprob = SHAPES[shape]
    cdt, sdt, out_dtype = dtypes(variant)
    ps, qss = weights(F, n, k, nprob, variant != "plain", sdt)
    seed = 1000 * m + n
    d = dict(n=n, k=k, m=m, nprob=nprob, cdt=cdt, sdt=sdt, out_dtype=out_dtype, packeds=ps, states=qss,
             xs=[make_act(m, k, seed=seed + i).to(cdt) for i in range(nprob)], biases=None, us=None, vs=None, scales=None)
    if variant.startswith("lora"):
        r = int(variant[4:])
        d["us"] = [make_act(m, r, seed=seed + 10 + i).to(cdt) for i in range(nprob)]
        d["vs"] = [make_weight(n, r, seed=seed + 20 + i, scale=0.05, dtype=cdt) for i in range(nprob)]
    if variant == "bias":
        d["biases"] = [make_weight(1, n, seed=seed + 30 + i, scale=0.5, dtype=cdt).view(-1) for i in range(nprob)]
    if variant == "row_scales":   # non-power-of-two scales; problem 1 unscaled
        gen = torch.Generator().manual_seed(seed + 40)
        d["scales"] = [None if i == 1 else (torch.rand(n, generator=gen) * 1.5 + 0.25).cuda() for i in range(nprob)]
    return d


def _pick(ts, order):
    return None if ts is None else [ts[i] for i in order]


def call(F, d, xs=None, order=None):
    """The grouped forward of `d` on the inputs `xs` (default: d's), over the problems in `order` (default: as given)."""
    order = list(range(d["nprob"])) if order is None else list(order)
    xs = d["xs"] if xs is None else xs
    return F.nf4_linear_group(False, [xs[i] for i in order], _pick(d["packeds"], order), _pick(d["states"], order),
                              _pick(d["biases"], order), _pick(d["us"], order), _pick(d["vs"], order),
                              out_dtype=d["out_dtype"], row_scales=_pick(d["scales"], order))


def call_single(F, d, i):
    """Problem i alone, with its own operands."""
    one = dict(d, nprob=1, **{key: None if d[key] is None else [d[key][i]]
                              for key in ("packeds", "states", "xs", "biases", "us", "vs", "scales")})
    return call(F, one)[0]


def path(names):
    """The GEMM path a call's kernel names show: 'skinny1' (the 1-token kernel), 'skinny', 'scratch', 'range' (the fused
    kernel without a split-K reduce) or 'splitk'."""
    if any("nf4_skinny_kernel_1tok" in s for s in names):
        return "skinny1"
    if any("nf4_skinny_kernel" in s for s in names):
        return "skinny"
    if any("nf4_scratch_gemm_kernel" in s for s in names):
        return "scratch"
    if any("nf4_gemm_wgmma_kernel" in s for s in names):
        return "splitk" if any("splitk_reduce" in s for s in names) else "range"
    return "none"


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32 if t.dtype == F32 else torch.int16).cpu().numpy()


def main(path_npz):
    import qlora_b200.functional as F
    from fused_kernel_names_case import kernel_names

    out = {}
    for case in CASES:
        cid = case_id(case)
        d = operands(F, case)
        call(F, d)   # warm-up: tensor maps, kernel attributes, schedules
        out[f"{cid}__names"] = np.array(kernel_names(lambda: call(F, d)))
        for i in range(d["nprob"]):
            call_single(F, d, i)
            out[f"{cid}__single{i}_names"] = np.array(kernel_names(lambda: call_single(F, d, i)))
            out[f"{cid}__single{i}"] = bits(call_single(F, d, i))
    torch.cuda.synchronize()
    np.savez(path_npz, **out)


if __name__ == "__main__":
    main(sys.argv[1])
