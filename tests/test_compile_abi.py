"""The custom ops torch.compile traces (qlora_b200/_ops.py), checked without a GPU: registration, schemas, and the fake
kernels' shape, dtype and stride rules on fake CUDA tensors, including the inputs they must reject before any launch."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import qlora_b200  # noqa: F401  (registers the ops)
import qlora_b200._ops  # noqa: F401

OPS = torch.ops.qlora_b200
BF16, F16, F32, U8 = torch.bfloat16, torch.float16, torch.float32, torch.uint8

SCHEMAS = {
    "nf4_linear_group": "qlora_b200::nf4_linear_group(bool is_bwd, Tensor[] inputs, Tensor[] packeds, Tensor[] absmax, "
                        "Tensor?[] code2, Tensor?[] absmax2, Tensor?[] offset, SymInt n_out, SymInt k_in, ScalarType state_dtype, "
                        "Tensor?[] biases, Tensor[] us, Tensor[] vs, Tensor(a13!)[] outs, ScalarType out_dtype, "
                        "Tensor?[] row_scales, Tensor(a16!)? w_scratch, bool return_scratch) -> Tensor",
    "lora_project": "qlora_b200::lora_project(Tensor x2d, Tensor lora_a, float scale) -> Tensor",
    "dequantize_nf4": "qlora_b200::dequantize_nf4(Tensor packed, Tensor absmax, Tensor? code2, Tensor? absmax2, Tensor? offset, "
                      "SymInt blocksize, SymInt blocksize2, Tensor(a7!) out) -> ()",
    "quantize_nf4": "qlora_b200::quantize_nf4(Tensor A, SymInt blocksize, Tensor(a2!) out, Tensor(a3!) absmax) -> ()",
    "quantize_blockwise": "qlora_b200::quantize_blockwise(Tensor code, Tensor A, SymInt blocksize, Tensor(a3!) out, "
                          "Tensor(a4!) absmax) -> ()",
    "dequantize_blockwise": "qlora_b200::dequantize_blockwise(Tensor code, Tensor A, Tensor absmax, SymInt blocksize, "
                            "Tensor(a4!) out) -> ()",
    "weight_row_norm2": "qlora_b200::weight_row_norm2(Tensor packed, Tensor absmax, Tensor? code2, Tensor? absmax2, "
                        "Tensor? offset, SymInt n_out, SymInt k_in, ScalarType dtype, SymInt blocksize, SymInt blocksize2) -> Tensor",
}


@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_op_is_registered_with_its_schema(name):
    op = getattr(OPS, name).default
    assert str(op._schema) == SCHEMAS[name]
    assert torch._C._dispatch_has_kernel_for_dispatch_key(op.name(), "Meta")   # the fake kernel


@pytest.fixture
def fake():
    with FakeTensorMode() as mode:
        yield mode


def _e(*shape, dtype=BF16):
    return torch.empty(*shape, dtype=dtype, device="cuda")


def _nested(n, k):
    return dict(absmax=[_e(n * k // 64, dtype=U8)], code2=[_e(256, dtype=F32)], absmax2=[_e(n * k // 64 // 256, dtype=F32)],
                offset=[_e((), dtype=F32)])


def _group(is_bwd=False, m=300, n=512, k=256, nprob=1, r=0, cdt=BF16, sdt=BF16, out_dtype=None, **over):
    st = _nested(n, k)
    c_in, f_out = (n, k) if is_bwd else (k, n)
    out_dtype = cdt if out_dtype is None else out_dtype
    args = dict(is_bwd=is_bwd, inputs=[_e(m, c_in, dtype=cdt)] * nprob, packeds=[_e(n * k // 2, 1, dtype=U8)] * nprob,
                absmax=st["absmax"] * nprob, code2=st["code2"] * nprob, absmax2=st["absmax2"] * nprob,
                offset=st["offset"] * nprob, n_out=n, k_in=k, state_dtype=sdt, biases=[],
                us=[_e(m, r, dtype=cdt)] * nprob if r else [], vs=[_e(*((r, k) if is_bwd else (n, r)), dtype=cdt)] * nprob if r else [],
                outs=[_e(m, f_out, dtype=out_dtype) for _ in range(1 if is_bwd else nprob)], out_dtype=out_dtype, row_scales=[],
                w_scratch=None, return_scratch=False)
    args.update(over)
    return args


@pytest.mark.parametrize("is_bwd,nprob,r,cdt,out_dtype", [
    (False, 1, 0, BF16, None), (False, 3, 64, BF16, F32), (False, 2, 136, BF16, F16), (True, 3, 64, BF16, None),
    (True, 1, 0, F16, F32), (False, 2, 8, F16, None)])
def test_group_fake_accepts(fake, is_bwd, nprob, r, cdt, out_dtype):
    scratch = OPS.nf4_linear_group(**_group(is_bwd=is_bwd, nprob=nprob, r=r, cdt=cdt, out_dtype=out_dtype))
    assert scratch.shape == (0,) and scratch.dtype == U8 and scratch.device.type == "cuda"


def test_group_fake_takes_pitched_outputs(fake):
    buf = _e(300, 520)
    OPS.nf4_linear_group(**_group(outs=[buf[:, :512]]))


def test_group_fake_scratch_size_is_decided_at_run_time():
    from torch.fx.experimental.symbolic_shapes import ShapeEnv

    with FakeTensorMode(shape_env=ShapeEnv()):
        scratch = OPS.nf4_linear_group(**_group(m=2048, return_scratch=True))
        assert isinstance(scratch.shape[0], torch.SymInt)


REJECTED = {
    "four_problems": dict(nprob=4),
    "fp32_inputs": dict(cdt=F32),
    "input_shape": dict(inputs=["x255"]),
    "bf16_output_under_fp16": dict(cdt=F16, out_dtype=BF16),
    "row_scales_with_fp16_state": dict(sdt=F16, row_scales=["scale"]),
    "row_scales_with_fp16_output": dict(out_dtype=F16, row_scales=["scale"]),
    "bias_in_dx": dict(is_bwd=True, biases=["bias"]),
    "lora_rank_mismatch": dict(r=64, us=["u32"]),
    "lent_output_dtype": dict(outs=["out_f32"]),
    "missing_output": dict(outs=[]),
    "output_shape": dict(outs=["out_wide"]),
    "mixed_quant_forms": dict(nprob=2, mixed=True),
    "u8_absmax_missing_code": dict(code2=[None]),
    "packed_size": dict(packeds=["short"]),
}


@pytest.mark.parametrize("case", sorted(REJECTED))
def test_group_fake_rejects(fake, case):
    over = dict(REJECTED[case])
    base = dict(nprob=over.pop("nprob", 1), cdt=over.pop("cdt", BF16), sdt=over.pop("sdt", BF16),
                out_dtype=over.pop("out_dtype", None), is_bwd=over.pop("is_bwd", False), r=over.pop("r", 0))
    args = _group(**base)
    subst = {"scale": _e(512, dtype=F32), "bias": _e(512), "u32": _e(300, 32), "out_f32": _e(300, 512, dtype=F32),
             "short": _e(100, 1, dtype=U8), "x255": _e(300, 255), "out_wide": _e(300, 520)}
    if over.pop("mixed", False):
        plain = _e(512 * 256 // 64, dtype=F32)
        args.update(absmax=[args["absmax"][0], plain], code2=[args["code2"][0], None], absmax2=[args["absmax2"][0], None],
                    offset=[args["offset"][0], None])
    for key, val in over.items():
        args[key] = [subst.get(v, v) if isinstance(v, str) else v for v in val] if isinstance(val, list) else val
    with pytest.raises((AssertionError, RuntimeError, ValueError)):
        OPS.nf4_linear_group(**args)


def test_ops_reject_cpu_tensors_before_any_launch():
    """The real kernels: host tensors are refused before the library is touched (no GPU needed to see it)."""
    x = torch.randn(4, 64, dtype=BF16)
    a = torch.randn(8, 64, dtype=BF16)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        OPS.lora_project(x, a, 1.0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        OPS.quantize_nf4(x.contiguous(), 64, torch.empty(128, 1, dtype=U8), torch.empty(4))


def test_lora_project_fake(fake):
    u = OPS.lora_project(_e(16, 1024), _e(136, 1024), 0.5)
    assert u.shape == (16, 136) and u.dtype == BF16
    assert OPS.lora_project(_e(2048, 1024), _e(64, 1024), 0.5).shape == (2048, 64)   # cuBLAS above 16 tokens
    with pytest.raises(AssertionError):
        OPS.lora_project(_e(4, 1024), _e(8, 512), 0.5)
    with pytest.raises(AssertionError):
        OPS.lora_project(_e(4, 1024), _e(8, 1024, dtype=F16), 0.5)


def test_quantization_fakes(fake):
    n, k = 512, 256
    st = _nested(n, k)
    packed = _e(n * k // 2, 1, dtype=U8)
    OPS.dequantize_nf4(packed, st["absmax"][0], st["code2"][0], st["absmax2"][0], st["offset"][0], 64, 256, _e(n, k))
    norm2 = OPS.weight_row_norm2(packed, st["absmax"][0], st["code2"][0], st["absmax2"][0], st["offset"][0], n, k, BF16, 64, 256)
    assert norm2.shape == (n,) and norm2.dtype == F32
    with pytest.raises(ValueError, match="blocksize"):
        OPS.dequantize_nf4(packed, st["absmax"][0], st["code2"][0], st["absmax2"][0], st["offset"][0], 96, 256, _e(n, k))
    with pytest.raises(ValueError, match="16/32-bit"):
        OPS.dequantize_nf4(packed, st["absmax"][0], st["code2"][0], st["absmax2"][0], st["offset"][0], 64, 256,
                           _e(n, k, dtype=U8))
    with pytest.raises(AssertionError):     # nested codes with an fp32 absmax
        OPS.dequantize_nf4(packed, _e(n * k // 64, dtype=F32), st["code2"][0], st["absmax2"][0], st["offset"][0], 64, 256,
                           _e(n, k))
    OPS.quantize_nf4(_e(n, k), 64, _e(n * k // 2, 1, dtype=U8), _e(n * k // 64, dtype=F32))
    with pytest.raises(AssertionError):     # absmax too short
        OPS.quantize_nf4(_e(n, k), 64, _e(n * k // 2, 1, dtype=U8), _e(8, dtype=F32))
    code = _e(256, dtype=F32)
    OPS.quantize_blockwise(code, _e(3000, dtype=F32), 256, _e(3000, dtype=U8), _e(12, dtype=F32))
    OPS.dequantize_blockwise(code, _e(3000, dtype=U8), _e(12, dtype=F32), 256, _e(3000, dtype=F32))
    with pytest.raises(AssertionError):     # codes and values swapped
        OPS.dequantize_blockwise(code, _e(3000, dtype=F32), _e(12, dtype=F32), 256, _e(3000, dtype=U8))
