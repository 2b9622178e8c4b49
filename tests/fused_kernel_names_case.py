"""Records which CUDA kernels the calls of tests/test_gpu_fused_edges.py::test_pitched_and_offset_outputs launch, for the dense
output and for every pitched or offset output view, and saves the kernel names as JSON to argv[1].  argv[2] and argv[3]
are the token counts that take the split-K and the range schedule at N x K.

The test runs this in a subprocess of its own.  A torch.profiler session tears CUPTI down when it ends, and CUPTI set up
again after that in a process that captures CUDA graphs is unreliable (torch turns the teardown off for its own CUDA-graph
paths for that reason): in the GPU suite, a later session then recorded no kernels at all.  Profiling here leaves the test
process as it was for the later suites that profile.  `operands`, `call` and `view` are shared with the test, so both sides
make the same calls; each view's base address modulo 16 is saved too, for the test to check that its views match."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gpu_helpers import make_act, make_weight  # noqa: E402

N, K = 4104, 4160
PITCH_PADS = (0, 4, 8)
OFFSETS = (0, 1, 2, 4, 8)
DTYPES = {"bf16": torch.bfloat16, "f32": torch.float32, "f16": torch.float16}
SENTINEL = -12345.0


def operands(F, m, is_bwd):
    """(packed, quant state, input, bias) of the N x K weight: a nested state, and a bias for the forward."""
    packed, qs = F.quantize_4bit(make_weight(N, K, seed=61), compress_statistics=True, quant_type="nf4")
    inp = make_act(m, N if is_bwd else K, seed=62)
    bias = None if is_bwd else make_weight(1, N, seed=63, scale=0.5).view(-1)
    return packed.t().contiguous(), qs, inp, bias


def call(F, ops, is_bwd, out_dtype, out=None):
    """The call under bf16 compute, writing `out` (None: a dense output it allocates); returns the output."""
    packed, qs, inp, bias = ops
    res = F.nf4_linear_group(is_bwd, [inp], [packed], [qs], None if bias is None else [bias], outs=None if out is None else [out],
                             out_dtype=out_dtype)
    return res if is_bwd else res[0]


def view(m, f_out, pad, off, dtype):
    """A flat buffer filled with the sentinel, and the [m, f_out] view into it at element offset `off` with row pitch
    f_out + pad."""
    ld = f_out + pad
    buf = torch.full((off + (m + 1) * ld,), torch.tensor(SENTINEL, dtype=dtype).item(), dtype=dtype, device="cuda")
    return buf, buf[off:off + m * ld].view(m, ld)[:, :f_out]


def key(schedule, is_bwd, dname, pad=None, off=None):
    return f"{schedule}-{'dx' if is_bwd else 'fwd'}-{dname}-" + ("dense" if pad is None else f"{pad}-{off}")


def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def main(path, m_splitk, m_range):
    import qlora_b200.functional as F

    names = {}
    for schedule, m in (("splitk", m_splitk), ("range", m_range)):
        for is_bwd in (False, True):
            ops = operands(F, m, is_bwd)
            f_out = K if is_bwd else N
            for dname, dtype in DTYPES.items():
                call(F, ops, is_bwd, dtype)   # warm-up: tensor maps, kernel attributes, schedules
                names[key(schedule, is_bwd, dname)] = kernel_names(lambda: call(F, ops, is_bwd, dtype))
                for pad in PITCH_PADS:
                    for off in OFFSETS:
                        _, out = view(m, f_out, pad, off, dtype)
                        k = key(schedule, is_bwd, dname, pad, off)
                        names[k] = kernel_names(lambda: call(F, ops, is_bwd, dtype, out))
                        names[k + "-base16"] = out.data_ptr() % 16
    with open(path, "w") as f:
        json.dump(names, f)


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]), int(sys.argv[3]))
