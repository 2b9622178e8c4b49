"""`bitsandbytes.functional` surface for the NF4 + double-quant path, on H100-native kernels.

Mirrors (names, argument meaning, return shapes, error behaviour) the upstream functions the
reference reaches through `qlora.py:15,249,318-326` (SURVEY.md 8b):

    quantize_4bit / dequantize_4bit           [upstream bitsandbytes/functional.py]
    quantize_blockwise / dequantize_blockwise [upstream bitsandbytes/functional.py]
    QuantState (+ as_dict/from_dict/to, list-style indexing)
    create_dynamic_map, create_normal_map, get_4bit_type

All device work goes through the C-ABI in include/qlora_b200.h (hand-written sm_90a CUDA).
CUDA tensors only: there is no CPU implementation in this package (the CPU restatement lives
in oracle/ and is test infrastructure).
"""
from __future__ import annotations

import json
from math import prod
from typing import Any, Optional

import torch
from torch import Tensor

from . import _lib, _ops
from ._lib import DTYPE_CODE, check, ptr, stream_ptr  # noqa: F401  (ptr, stream_ptr: used by callers of F)

name2qmap: dict[str, Tensor] = {}

# Bookkeeping used by bench.py: number of launches of OUR kernels, and (when set to a list) CUDA-event
# pairs recorded on the launching stream around every fused-GEMM launch: (kind, M, N, K, start, end).
LAUNCH_COUNTER = [0]
EVENT_LOG = None

# A.1 — NF4 codebook (normalised N(0,1) quantiles, offset 0.9677083); fp32-exact literals.
_NF4_VALUES = [
    -1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453,
    -0.28444138169288635, -0.18477343022823334, -0.09105003625154495, 0.0,
    0.07958029955625534, 0.16093020141124725, 0.24611230194568634, 0.33791524171829224,
    0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0,
]


def create_normal_map(offset: float = 0.9677083, use_extra_value: bool = True) -> Tensor:
    """NF4 data type as a 256-entry map (16 used values, zero padded), like upstream."""
    if not use_extra_value:
        raise NotImplementedError("only the asymmetric NF4 map (use_extra_value=True) is implemented")
    values = torch.tensor(_NF4_VALUES, dtype=torch.float32)
    return torch.cat([values, torch.zeros(256 - 16)])


def create_dynamic_map(signed: bool = True, max_exponent_bits: int = 7, total_bits: int = 8) -> Tensor:
    """Dynamic-tree 8-bit codebook used for the second-level (double) quantization of absmax.

    Follows upstream's construction order exactly (torch fp32 linspace -> midpoint means ->
    scale by 10**(i - max_exponent_bits + 1) -> append 0 and 1 -> sort) so the 256 fp32 values
    are the ones checkpoints quantized by bitsandbytes carry.
    """
    data: list[float] = []
    non_sign_bits = total_bits - 1
    additional_items = 2 ** (non_sign_bits - max_exponent_bits) - 1
    i = 0
    for i in range(max_exponent_bits):
        exp = i + non_sign_bits - max_exponent_bits
        fraction_items = int(2**exp + 1 if signed else 2 ** (exp + 1) + 1)
        boundaries = torch.linspace(0.1, 1, fraction_items)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    if additional_items > 0:
        boundaries = torch.linspace(0.1, 1, additional_items + 1)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    data.append(0)
    data.append(1.0)
    assert len(data) == 2**total_bits
    data += [0] * (256 - len(data))
    data.sort()
    return torch.tensor(data, dtype=torch.float32)


def get_4bit_type(typename: str, device=None, blocksize: int = 64) -> Tensor:
    if device is None:
        device = "cuda"
    if typename == "nf4":
        key = f"nf4@{torch.device(device)}"
        if key not in name2qmap:  # cached per device: building it is a synchronous H2D copy
            name2qmap[key] = torch.tensor(_NF4_VALUES, dtype=torch.float32, device=device)
        return name2qmap[key].clone()
    if typename == "fp4":
        raise NotImplementedError("quant_type='fp4' is outside this build's scope (NF4 only; SURVEY.md 2.2)")
    raise NotImplementedError(f"Typename {typename} not supported")


def set_quant_math(mode: str) -> None:
    """Arithmetic of the quantizers' reciprocal-and-scale: "ieee" (default; bit-exact with the CPU oracle) or "approx"
    (`rcp.approx.ftz` + `mul.ftz`: what upstream's `--use_fast_math` build executes; SURVEY.md A.5(i)).  Process-wide."""
    if mode not in ("ieee", "approx"):
        raise ValueError("quant math mode must be 'ieee' or 'approx'")
    check(_lib.load().qb200_set_quant_math(1 if mode == "approx" else 0), "set_quant_math")


def get_quant_math() -> str:
    return "approx" if _lib.load().qb200_get_quant_math() else "ieee"


def _pack_dict_to_tensor(source_dict: dict[str, Any]) -> Tensor:
    blob = json.dumps(source_dict).encode("utf-8")
    return torch.frombuffer(bytearray(blob), dtype=torch.uint8).clone()


def _unpack_tensor_to_dict(tensor_data: Tensor) -> dict[str, Any]:
    return json.loads(bytes(tensor_data.cpu().numpy().tobytes()).decode("utf-8"))


class QuantState:
    """Container for the quantization state of a (possibly double-quantized) tensor.

    Same constructor, attributes, list-style indexing and (un)packing as upstream's
    `bitsandbytes.functional.QuantState` (SURVEY.md 8a row a6).
    """

    valid_quant_types = ("fp4", "nf4")
    valid_qs_type_keys = [f"bitsandbytes__{x}" for x in valid_quant_types]
    valid_qs_keys = [
        "absmax", "quant_map", "nested_absmax", "nested_quant_map", "quant_state", "quant_type",
        "blocksize", "dtype", "shape", "nested_blocksize", "nested_dtype", "nested_offset",
    ]

    def __init__(self, absmax, shape=None, code=None, blocksize=None, quant_type=None, dtype=None, offset=None, state2=None):
        self.absmax = absmax
        self.shape = shape
        self.code = code
        self.dtype = dtype
        self.blocksize = blocksize
        self.quant_type = quant_type
        self.offset = offset
        self.state2 = state2
        self.nested = state2 is not None

    def __getitem__(self, idx):
        # 0.40-era call sites unpack the state as a list
        if self.nested:
            list_repr = [self.absmax, self.shape, self.dtype, self.blocksize, [self.offset, self.state2], self.quant_type]
        else:
            list_repr = [self.absmax, self.shape, self.dtype, self.blocksize, None, self.quant_type]
        return list_repr[idx]

    @classmethod
    def from_dict(cls, qs_dict: dict[str, Any], device) -> "QuantState":
        qs_dict = dict(qs_dict)
        qs_key = [k for k, v in qs_dict.items() if "quant_state" in k and isinstance(v, Tensor)]
        if not len(qs_key) and "quant_type" not in qs_dict:
            raise ValueError("Expected packed or unpacked quant_state items, found neither")
        elif len(qs_key) > 1 or (len(qs_key) == 1 and qs_key[0].split(".")[-1] not in cls.valid_qs_type_keys):
            raise ValueError(f"There should be exactly one `quant_state` item with ending from {cls.valid_qs_type_keys}.\nDetected {qs_key}.")
        if len(qs_key) == 1:
            qs_dict.update(_unpack_tensor_to_dict(qs_dict.pop(qs_key[0])))
        qs_dict = {k.split(".")[-1]: v for k, v in qs_dict.items()}
        assert set(qs_dict.keys()).issubset(cls.valid_qs_keys), f"unexpected quant-state keys {set(qs_dict) - set(cls.valid_qs_keys)}"

        if "nested_absmax" in qs_dict:
            offset = torch.tensor(float(qs_dict["nested_offset"])).to(device)
            state2 = cls(
                absmax=qs_dict["nested_absmax"].to(device),
                blocksize=qs_dict["nested_blocksize"],
                code=qs_dict["nested_quant_map"].to(device),
                dtype=getattr(torch, qs_dict["nested_dtype"]),
            )
        else:
            offset, state2 = None, None
        return cls(
            quant_type=qs_dict["quant_type"],
            absmax=qs_dict["absmax"].to(device),
            blocksize=qs_dict["blocksize"],
            code=qs_dict["quant_map"].to(device),
            dtype=getattr(torch, qs_dict["dtype"]),
            shape=torch.Size(qs_dict["shape"]) if qs_dict["shape"] is not None else None,
            offset=offset,
            state2=state2,
        )

    def as_dict(self, packed: bool = False) -> dict[str, Any]:
        qs_dict: dict[str, Any] = {
            "quant_type": self.quant_type,
            "absmax": self.absmax,
            "blocksize": self.blocksize,
            "quant_map": self.code,
            "dtype": str(self.dtype).replace("torch.", ""),
            "shape": tuple(self.shape) if self.shape is not None else None,
        }
        if self.nested:
            qs_dict.update(
                {
                    "nested_absmax": self.state2.absmax,
                    "nested_blocksize": self.state2.blocksize,
                    "nested_quant_map": self.state2.code.clone(),
                    "nested_dtype": str(self.state2.dtype).replace("torch.", ""),
                    "nested_offset": self.offset.item(),
                }
            )
        if not packed:
            return qs_dict
        qs_packed = {k: v for k, v in qs_dict.items() if isinstance(v, Tensor)}
        non_tensor = {k: v for k, v in qs_dict.items() if not isinstance(v, Tensor)}
        qs_packed["quant_state." + "bitsandbytes__" + self.quant_type] = _pack_dict_to_tensor(non_tensor)
        return qs_packed

    def to(self, device):
        self.code = self.code.to(device) if self.code is not None else None
        self.absmax = self.absmax.to(device)
        if self.nested:
            self.offset = self.offset.to(device)
            self.state2.absmax = self.state2.absmax.to(device)
            self.state2.code = self.state2.code.to(device)
        return self

    def __eq__(self, other):
        if not isinstance(other, QuantState):
            return False
        return (
            torch.allclose(self.absmax, other.absmax, atol=1e-6)
            and self.shape == other.shape
            and torch.allclose(self.code, other.code, atol=1e-6)
            and self.dtype == other.dtype
            and self.blocksize == other.blocksize
            and self.quant_type == other.quant_type
            and (self.offset == other.offset if self.offset is not None and other.offset is not None else self.offset is other.offset)
            and (self.state2 == other.state2 if self.state2 is not None and other.state2 is not None else self.state2 is other.state2)
        )

    __hash__ = None  # mutable container


def _default_code(device) -> Tensor:
    if "dynamic" not in name2qmap:
        name2qmap["dynamic"] = create_dynamic_map()
    key = f"dynamic@{device}"
    if key not in name2qmap:
        name2qmap[key] = name2qmap["dynamic"].to(device)
    return name2qmap[key]


def quantize_blockwise(A: Tensor, code: Optional[Tensor] = None, absmax: Optional[Tensor] = None, out: Optional[Tensor] = None,
                       blocksize: int = 4096, nested: bool = False) -> tuple[Tensor, QuantState]:
    """8-bit blockwise quantization against a 256-entry codebook (K2; used for nested absmax)."""
    dev = _ops._device(A)
    if code is None:
        code = _default_code(dev)
    code = code.to(device=dev, dtype=torch.float32).contiguous()
    _ops._check_blocksize(blocksize)
    n = A.numel()
    blocks = -(n // -blocksize)
    if absmax is None:
        absmax = torch.empty((blocks,), device=dev, dtype=torch.float32)  # fully written by the kernel
    if out is None:
        out = torch.empty(A.shape, dtype=torch.uint8, device=dev)  # always contiguous (empty_like would keep A's strides)
    elif not out.is_contiguous() or out.dtype != torch.uint8 or out.numel() != n:
        raise ValueError("quantize_blockwise: `out` must be a contiguous uint8 tensor with A.numel() elements")
    A32 = A.contiguous().float()  # widening is exact; the kernel computes in fp32 like upstream
    _ops.quantize_blockwise(code, A32, blocksize, out, absmax)
    if nested:
        offset = absmax.mean()
        absmax -= offset
        qabsmax, state2 = quantize_blockwise(absmax, blocksize=blocksize, nested=False)
        state = QuantState(absmax=qabsmax, code=code, blocksize=blocksize, dtype=A.dtype, offset=offset, state2=state2)
    else:
        state = QuantState(absmax=absmax, code=code, blocksize=blocksize, dtype=A.dtype)
    return out, state


def dequantize_blockwise(A: Tensor, quant_state: Optional[QuantState] = None, absmax: Optional[Tensor] = None,
                         code: Optional[Tensor] = None, out: Optional[Tensor] = None, blocksize: int = 4096,
                         nested: bool = False) -> Tensor:
    """8-bit blockwise dequantization (K3): out[i] = code[A[i]] * absmax[i // blocksize]."""
    assert quant_state is not None or absmax is not None
    dev = _ops._device(A)
    if quant_state is None:
        if code is None:
            code = _default_code(dev)
        quant_state = QuantState(absmax=absmax, code=code, blocksize=blocksize, dtype=torch.float32)
    absmax = quant_state.absmax
    if quant_state.nested:
        absmax = dequantize_blockwise(quant_state.absmax, quant_state.state2)
        absmax = absmax + quant_state.offset
    if absmax.dtype != torch.float32:
        absmax = absmax.float()
    _ops._check_blocksize(quant_state.blocksize)
    code32 = quant_state.code.to(device=dev, dtype=torch.float32).contiguous()
    out32 = out if (out is not None and out.dtype == torch.float32) else torch.empty(A.shape, dtype=torch.float32, device=dev)
    _ops.dequantize_blockwise(code32, A.contiguous(), absmax.contiguous(), quant_state.blocksize, out32)
    target = quant_state.dtype if quant_state.dtype is not None else torch.float32
    if out is not None and out is not out32:
        out.copy_(out32)
        return out
    return out32 if target == torch.float32 else out32.to(target)


def quantize_4bit(A: Tensor, absmax: Optional[Tensor] = None, out: Optional[Tensor] = None, blocksize: int = 64,
                  compress_statistics: bool = False, quant_type: str = "fp4", quant_storage=torch.uint8) -> tuple[Tensor, QuantState]:
    """NF4 blockwise quantization (K1 [+ K2 when compress_statistics]).

    Returns (packed uint8 tensor of shape [(n+1)//2, 1], QuantState).  Even element in the high
    nibble; absmax per `blocksize` flat elements; with `compress_statistics` the fp32 absmax is
    itself quantized to 8 bits in blocks of 256 after subtracting its mean (double quantization).
    """
    dev = _ops._device(A)
    if quant_type not in ("fp4", "nf4"):
        raise NotImplementedError(f"4-bit quantization data type {quant_type} is not implemented.")
    if quant_type == "fp4":
        raise NotImplementedError("quant_type='fp4' is outside this build's scope (NF4 only; SURVEY.md 2.2)")
    if A.dtype not in DTYPE_CODE:
        raise ValueError(f"Blockwise quantization only supports 16/32-bit floats, but got {A.dtype}")
    _ops._check_blocksize(blocksize)
    if quant_storage != torch.uint8:
        raise NotImplementedError("quant_storage other than torch.uint8 is not implemented")
    n = A.numel()
    input_shape = A.shape
    blocks = -(n // -blocksize)
    if absmax is None:
        absmax = torch.empty((blocks,), device=dev, dtype=torch.float32)  # fully written by the kernel
    if out is None:
        out = torch.empty(((n + 1) // 2, 1), dtype=torch.uint8, device=dev)
    A = A.contiguous()
    _ops.quantize_nf4(A, blocksize, out, absmax)
    code = get_4bit_type(quant_type, device=dev)
    if compress_statistics:
        offset = absmax.mean()  # reduction order = torch's, exactly as the reference computes it
        absmax -= offset
        qabsmax, state2 = quantize_blockwise(absmax, blocksize=256)
        del absmax
        state = QuantState(absmax=qabsmax, shape=input_shape, dtype=A.dtype, blocksize=blocksize, code=code,
                           quant_type=quant_type, offset=offset, state2=state2)
    else:
        state = QuantState(absmax=absmax, shape=input_shape, dtype=A.dtype, blocksize=blocksize, code=code, quant_type=quant_type)
    return out, state


def dequantize_4bit(A: Tensor, quant_state: Optional[QuantState] = None, absmax: Optional[Tensor] = None,
                    out: Optional[Tensor] = None, blocksize: int = 64, quant_type: str = "fp4") -> Tensor:
    """NF4 dequantization (K4; for nested states K3 + offset add + K4 run as ONE kernel).

    Returns a tensor of `quant_state.shape` / `quant_state.dtype`; like upstream, if `A` is the
    transposed `[1, n/2]` view that `matmul_4bit` passes, the result is returned transposed.
    """
    dev = _ops._device(A)
    if quant_state is None:
        assert absmax is not None and out is not None
        if quant_type != "nf4":
            raise NotImplementedError("quant_type='fp4' is outside this build's scope (NF4 only; SURVEY.md 2.2)")
        quant_state = QuantState(absmax=absmax, shape=out.shape, dtype=out.dtype, blocksize=blocksize, quant_type=quant_type)
    if quant_state.quant_type != "nf4":
        raise NotImplementedError(f"4-bit quantization data type {quant_state.quant_type} is not implemented.")
    _ops._check_blocksize(quant_state.blocksize)
    if out is None:
        out = torch.empty(quant_state.shape, dtype=quant_state.dtype, device=dev)
    if out.dtype not in DTYPE_CODE:
        raise ValueError(f"Blockwise quantization only supports 16/32-bit floats, but got {out.dtype}")
    packed = A if A.is_contiguous() else A.contiguous()  # the [1, n/2] .t() view of a [n/2, 1] tensor is contiguous
    _ops.dequantize_nf4(packed, *_state_args(quant_state, dev), out)
    is_transposed = A.shape[0] == 1
    return out.t() if is_transposed else out


def quantize_nf4(A, absmax=None, out=None, blocksize=64, compress_statistics=False, quant_storage=torch.uint8):
    return quantize_4bit(A, absmax, out, blocksize, compress_statistics, "nf4", quant_storage)


def dequantize_nf4(A, quant_state=None, absmax=None, out=None, blocksize=64):
    return dequantize_4bit(A, quant_state, absmax, out, blocksize, "nf4")


# --------------------------------------------------------------------------------------
# Fused linear entry points (new exports; SURVEY.md 8b "New export for the fused path")
# --------------------------------------------------------------------------------------

# Quant-state dtypes for which the fused kernels read exactly `dequantize_4bit(...).to(compute_dtype)`, per fused compute
# dtype: the product table T16_rn(LUT[j] * absmax) for a bf16 or fp32 state under bf16 compute and for an fp16 or fp32 state
# under fp16 compute, and the double-rounded table bf16_rn(fp16_rn(LUT[j] * absmax)) for an fp16 state under bf16 compute.
# A bf16 state under fp16 compute stays on the unfused path: no kernel table rounds bf16, then fp16.
_FUSED_STATE_DTYPES = {torch.bfloat16: (torch.bfloat16, torch.float16, torch.float32), torch.float16: (torch.float16, torch.float32)}


def fused_supported(quant_state: QuantState, compute_dtype: torch.dtype) -> bool:
    """Shapes/dtypes the fused wgmma kernel handles; everything else takes the unfused GPU path."""
    if quant_state.quant_type != "nf4" or quant_state.blocksize != 64:
        return False
    if (quant_state.shape is None or len(quant_state.shape) != 2
            or quant_state.dtype not in _FUSED_STATE_DTYPES.get(compute_dtype, ())):
        return False
    n_out, k_in = quant_state.shape
    if k_in % 64 != 0 or n_out % 8 != 0:
        return False
    if quant_state.nested and quant_state.state2.blocksize != 256:
        return False
    return True


def double_rounded(quant_state: QuantState, compute_dtype: torch.dtype) -> bool:
    """Whether the fused kernels round this state's weights twice, bf16_rn(fp16_rn(LUT[j] * absmax)): an fp16 state under
    bf16 compute.  Problems of one grouped launch agree on it."""
    return compute_dtype == torch.bfloat16 and quant_state.dtype == torch.float16


def as_compute_2d(t: Tensor, dtype: torch.dtype = torch.bfloat16) -> Tensor:
    """`t` as the contiguous [rows, last dim] matrix of the compute dtype (bf16 or fp16) the fused kernels read (cast and
    copied only where needed)."""
    t2 = t.reshape(-1, t.shape[-1])
    if t2.dtype != dtype:
        t2 = t2.to(dtype)
    return t2 if t2.is_contiguous() else t2.contiguous()


def out_dtype_for(in_dtype: torch.dtype, compute_dtype: torch.dtype = torch.bfloat16) -> torch.dtype:
    """What a fused launch writes for activations of `in_dtype`: fp32 for fp32 (the kernel's epilogue widens the result
    rounded to the compute dtype, as `Linear4bit.forward` returns fp32 for fp32 input), fp16 for fp16 under bf16 compute
    (the bf16-rounded result rounded to fp16), else the compute dtype."""
    if in_dtype == torch.float32 or (in_dtype == torch.float16 and compute_dtype == torch.bfloat16):
        return in_dtype
    return compute_dtype


def _event_begin():
    LAUNCH_COUNTER[0] += 1
    if EVENT_LOG is None:
        return None
    ev = torch.cuda.Event(enable_timing=True)
    ev.record()
    return ev


def _event_end(kind, m, n, k, ev):
    if ev is not None:
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        EVENT_LOG.append((kind, m, n, k, ev, ev1))


def _checked(t: Tensor, dtype: torch.dtype, dev: torch.device, what: str) -> Tensor:
    """A state tensor as the kernels read it: `dtype`, contiguous, on the activation's GPU.  A state that a loader cast
    (e.g. `torch_dtype` applied to absmax) or left on another device is converted / moved here instead of being read as
    raw bytes; the converted copy is cached on the QuantState by the caller."""
    if t is None:
        raise RuntimeError(f"quant_state.{what} is missing")
    if t.device != dev or t.dtype != dtype or not t.is_contiguous():
        t = t.to(device=dev, dtype=dtype).contiguous()
    return t


def _state_tensors(qs: QuantState, dev: torch.device):
    """(absmax_u8, code256, absmax2, offset, absmax_f32) validated for the fused kernel (ADVICE r1: dtype / device /
    contiguity are checked, never assumed).  Only converted copies are written back, so a state the kernels can read as it
    is stays untouched (what lets torch.compile trace this without a side effect)."""
    if qs.nested:
        s2 = qs.state2
        for obj, name, dtype, what in ((qs, "absmax", torch.uint8, "absmax"), (s2, "code", torch.float32, "state2.code"),
                                       (s2, "absmax", torch.float32, "state2.absmax"), (qs, "offset", torch.float32, "offset")):
            t = getattr(obj, name)
            c = _checked(t, dtype, dev, what)
            if c is not t:
                setattr(obj, name, c)
        return qs.absmax, s2.code, s2.absmax, qs.offset, None
    a = _checked(qs.absmax, torch.float32, dev, "absmax")
    if a is not qs.absmax:
        qs.absmax = a
    return None, None, None, None, qs.absmax


def _state_args(qs: QuantState, dev: torch.device):
    """The state as the dequantize ops take it: (absmax, code2, absmax2, offset, blocksize, blocksize2)."""
    if qs.nested:
        a_u8, code, a2, off, _ = _state_tensors(qs, dev)
        return a_u8, code, a2, off, qs.blocksize, qs.state2.blocksize
    return _checked(qs.absmax, torch.float32, dev, "absmax"), None, None, None, qs.blocksize, 0



def nf4_linear_group(is_bwd: bool, inputs, packeds, states, biases=None, us=None, vs=None, outs=None,
                     out_dtype: Optional[torch.dtype] = None, row_scales=None, w_scratch: Optional[Tensor] = None,
                     return_scratch: bool = False):
    """1..3 `Linear4bit` of one shape in ONE launch of the fused kernel (`qb200_nf4_linear_group_reuse`, or
    `qb200_nf4_linear_group_typed` with row scales), through the `qlora_b200::nf4_linear_group` op.

    The inputs' dtype (bf16 or fp16) is the compute dtype: U / V / bias are of it too and `out_dtype` is it (the default) or
    fp32 (the result rounded to it, widened); under bf16 compute it may also be fp16 (the bf16-rounded result rounded to
    fp16).  The states share one dtype, which selects the weights: those of `dequantize_4bit(...).to(compute dtype)`.
    Event-log kinds end in `_f16` for fp16 compute, and in `_sf16` and / or `_of16` for bf16 compute over an fp16 state or
    with an fp16 output.

    forward  (is_bwd=False): out_p = in_p . W_p^T (+bias_p) + U_p . V_p^T for every problem (the inputs may be one tensor);
                             returns the list of outputs.
    backward (is_bwd=True) : ONE output  sum_p (in_p . W_p + U_p . V_p), accumulated in the kernel; returns it.
    Inputs / U / outputs may be column slices of wider row-major buffers (row pitch passed through).
    row_scales: None, or one fp32 [N] tensor (or None) per problem; W_p is then diag(row_scales[p]) . W_p, the scale folded
    into the absmax of every NF4 block of the row.
    Training token counts (the scratch path) dequantize every W_p into a bf16 scratch that the GEMM reads.  return_scratch:
    also return that scratch, or None when the call left no W_p there: (result, scratch).  w_scratch: a scratch returned by
    an earlier call on the same packed weights and states, in the same order; a call that takes the scratch path then skips
    the dequantize launches and reads it.  Under torch.compile no scratch is returned (None): whether a call leaves one is
    decided at run time, and a graph cannot branch on it.
    """
    n = len(states)
    assert 1 <= n <= 3 and len(inputs) == n and len(packeds) == n
    dev = _ops._device(*inputs, *packeds)
    n_out, k_in = states[0].shape
    for qs in states:
        assert tuple(qs.shape) == (n_out, k_in), "grouped problems must share their weight shape"
    cdt = inputs[0].dtype
    twice = double_rounded(states[0], cdt)
    assert all(double_rounded(qs, cdt) == twice for qs in states), "grouped problems must share the rounding of their weights"
    sts = [_state_tensors(qs, dev) for qs in states]
    return_scratch_op = return_scratch and not torch.compiler.is_compiling()
    out_dtype = cdt if out_dtype is None else out_dtype
    if outs is None:
        m, f_out = inputs[0].shape[0], (k_in if is_bwd else n_out)
        outs = [torch.empty((m, f_out), dtype=out_dtype, device=dev) for _ in range(1 if is_bwd else n)]
    scratch = _ops.nf4_linear_group(
        is_bwd, list(inputs), list(packeds), [a_f32 if a_u8 is None else a_u8 for a_u8, _, _, _, a_f32 in sts],
        [t[1] for t in sts], [t[2] for t in sts], [t[3] for t in sts], n_out, k_in, states[0].dtype,
        [] if biases is None else list(biases), [] if us is None else list(us), [] if vs is None else list(vs),
        list(outs), out_dtype,
        [] if row_scales is None else list(row_scales), w_scratch, return_scratch_op)
    res = outs[0] if is_bwd else list(outs)
    if return_scratch:
        if not return_scratch_op or scratch.numel() == 0:
            return res, None
        return res, (scratch if w_scratch is None else w_scratch)
    return res


def scratch_to_save(scratch: Optional[Tensor], needs_dx: bool) -> list:
    """What an autograd forward saves so that its dX launch can reuse the forward's bf16 weight copy (`nf4_linear_group`'s
    scratch): nothing when the call left none or no dX will run; the copy itself in a forward that runs inside a backward
    (a gradient-checkpoint recompute, whose dX follows within the same layer's backward); else a one-byte placeholder of its
    shape, so that a forward outside backward never holds a copy.  Checkpointing requires the original forward and its
    recompute to save tensors of equal shape, dtype and device, and only the recompute's saved tensors reach the backward
    (the recompute's ctx is discarded), so the copy has to travel through `save_for_backward`."""
    if scratch is None or not needs_dx:
        return []
    if torch._C._current_graph_task_id() != -1:
        return [scratch]
    return [scratch.new_empty(1).expand(scratch.shape)]


def saved_scratch(saved) -> Optional[Tensor]:
    """The weight copy `scratch_to_save` put last among the saved tensors, or None for its placeholder."""
    t = saved[-1]
    return t if t.stride(0) == 1 else None


def _linear_ex(is_bwd: bool, inp: Tensor, packed: Tensor, quant_state: QuantState, bias: Optional[Tensor] = None,
               u: Optional[Tensor] = None, v: Optional[Tensor] = None, out_dtype: Optional[torch.dtype] = None) -> Tensor:
    """One Linear4bit through the fused kernel (+ the split-K reduce when the schedule asks for a workspace)."""
    res = nf4_linear_group(is_bwd, [inp], [packed], [quant_state], None if bias is None else [bias],
                           None if u is None else [u], None if v is None else [v], out_dtype=out_dtype)
    return res if is_bwd else res[0]


def nf4_linear_fwd(x2d: Tensor, packed: Tensor, quant_state: QuantState, bias: Optional[Tensor] = None,
                   out_dtype: Optional[torch.dtype] = None) -> Tensor:
    """Y[M,N] = X[M,K] . W^T (+bias) straight from the packed NF4 state (fused kernel); X bf16 or fp16, Y of X's dtype (or
    `out_dtype` fp32)."""
    return _linear_ex(False, x2d, packed, quant_state, bias, out_dtype=out_dtype)


def nf4_linear_bwd_dx(dy2d: Tensor, packed: Tensor, quant_state: QuantState, out_dtype: Optional[torch.dtype] = None) -> Tensor:
    """dX[M,K] = dY[M,N] . W straight from the packed NF4 state (same kernel, W consumed MN-major)."""
    return _linear_ex(True, dy2d, packed, quant_state, out_dtype=out_dtype)


LORA_MAX_RANK = 256


def lora_fused_supported(quant_state: QuantState, compute_dtype: torch.dtype, r: int) -> bool:
    """Whether the fused kernels take a LoRA term of rank r over this state: r a multiple of 8 (16-byte TMA rows) up to
    256, contracted in one 64-wide step per 64 ranks (one 64-rank chunk of the epilogue on the skinny kernels)."""
    return fused_supported(quant_state, compute_dtype) and 8 <= r <= LORA_MAX_RANK and r % 8 == 0


def nf4_linear_fwd_lora(x2d: Tensor, packed: Tensor, quant_state: QuantState, u: Tensor, v: Tensor,
                        bias: Optional[Tensor] = None, out_dtype: Optional[torch.dtype] = None) -> Tensor:
    """Y[M,N] = X . W^T (+bias) + U . V^T in one launch (U[M,r], V[N,r] = lora_B.weight, of X's dtype)."""
    return _linear_ex(False, x2d, packed, quant_state, bias, u, v, out_dtype=out_dtype)


LORA_PROJECT_MAX_TOKENS = 16


def lora_project(x2d: Tensor, lora_a: Tensor, scale: float) -> Tensor:
    """U[M,r] = scale * x2d . lora_a^T for at most 16 tokens (`qb200_lora_project`): the lora_A projection of a decode step.
    bf16 (or fp16: `qb200_lora_project_typed`) operands of one dtype, fp32 sum, one rounding — what
    `torch.addmm(..., alpha=scale)` returns, in one 3 us launch that chains with the skinny kernel by programmatic dependent
    launch."""
    m, k = x2d.shape
    assert 1 <= m <= LORA_PROJECT_MAX_TOKENS and lora_a.shape[1] == k and k % 8 == 0
    assert x2d.dtype in (torch.bfloat16, torch.float16) and lora_a.dtype == x2d.dtype
    return _ops.lora_project(x2d, lora_a if lora_a.is_contiguous() else lora_a.contiguous(), float(scale))


def nf4_linear_bwd_dx_lora(dy2d: Tensor, packed: Tensor, quant_state: QuantState, u: Tensor, vt: Tensor,
                           out_dtype: Optional[torch.dtype] = None) -> Tensor:
    """dX[M,K] = dY . W + U . Vt in one launch (U[M,r], Vt[r,K] = lora_A.weight, of dY's dtype)."""
    return _linear_ex(True, dy2d, packed, quant_state, None, u, vt, out_dtype=out_dtype)


# --------------------------------------------------------------------------------------
# DoRA over the NF4 base (weight-decomposed LoRA, Liu et al. 2024): the row norm of W + s.B.A without materialising W
# --------------------------------------------------------------------------------------

def weight_row_norm2(packed: Tensor, quant_state: QuantState) -> Tensor:
    """||W_f||^2 for every row f of the frozen NF4 weight: the bf16 weight `dequantize_4bit` returns, squared and summed in
    fp32; fp32 [N].  Cached on the QuantState (the base never changes), so call it once at setup: inside a CUDA-graph
    capture a missing cache is an error, not a lazy allocation."""
    cached = getattr(quant_state, "row_norm2", None)
    if cached is not None:
        return cached
    compiling = torch.compiler.is_compiling()
    if not compiling and torch.cuda.is_current_stream_capturing():
        raise RuntimeError("weight_row_norm2: compute the row norms of a frozen base before capturing a CUDA graph")
    if quant_state.quant_type != "nf4":
        raise NotImplementedError(f"4-bit quantization data type {quant_state.quant_type} is not implemented.")
    n_out, k_in = quant_state.shape
    packed = packed if packed.is_contiguous() else packed.contiguous()
    norm2 = _ops.weight_row_norm2(packed, *_state_args(quant_state, _ops._device(packed))[:4], n_out, k_in, quant_state.dtype,
                                  quant_state.blocksize, quant_state.state2.blocksize if quant_state.nested else 0)
    if not compiling:   # a traced graph cannot store into the state: it computes the norms on every call without a cache
        quant_state.row_norm2 = norm2
    return norm2


def dora_weight_norm(packeds, states, lora_as, lora_bs, scaling: float):
    """DoRA's weight norm n_f = ||W_f + s (B A)_f||_2 (fp32 [N], no gradient) for 1..3 frozen NF4 weights of one shape,
    from the expansion
        n^2 = ||W_f||^2 + 2 s sum_j B[f, j] P[j, f] + s^2 (B G B^T)_ff,   P = A . W^T [r, N],  G = A . A^T [r, r],
    with ||W_f||^2 cached per base (`weight_row_norm2`), P from ONE launch of the fused forward with the adapters A_p as r-token
    inputs, and the rest small fp32 ops.  Single tensors or lists (q/k/v, gate/up) are accepted; returns the same form."""
    single = isinstance(states, QuantState)
    if single:
        packeds, states, lora_as, lora_bs = [packeds], [states], [lora_as], [lora_bs]
    with torch.no_grad():
        ps = nf4_linear_group(False, [a.detach() for a in lora_as], list(packeds), list(states), out_dtype=torch.float32)
        norms = []
        for packed, qs, a, b, p in zip(packeds, states, lora_as, lora_bs, ps):
            a32, b32 = a.detach().float(), b.detach().float()
            cross = (b32 * p.t()).sum(1)
            quad = ((b32 @ (a32 @ a32.t())) * b32).sum(1)
            n2 = weight_row_norm2(packed, qs) + (2.0 * scaling) * cross + (scaling * scaling) * quad
            norms.append(n2.clamp_min_(0.0).sqrt_())
    return norms[0] if single else norms
