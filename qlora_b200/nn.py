"""`bitsandbytes.nn` surface: Linear4bit / Params4bit (+ NF4/FP4 aliases and 8-bit name stubs).

What the reference and its callers rely on (SURVEY.md 8b):
  * qlora.py:249   `isinstance(module, bnb.nn.Linear4bit)` collects LoRA targets;
  * transformers    `Linear4bit(in, out, bias, compute_dtype, compress_statistics=..., quant_type=...)`,
                    `Params4bit(value, requires_grad=False, **old.__dict__).to(device)`,
                    `Params4bit.from_prequantized(data, quantized_stats, ...)`;
  * peft            reads `.compute_dtype`, `.weight.compress_statistics`, `.weight.quant_type`;
  * state dict keys `weight`, `weight.absmax`, `weight.quant_map`, `weight.nested_absmax`,
                    `weight.nested_quant_map`, `weight.quant_state.bitsandbytes__nf4`.
"""
from __future__ import annotations

import copy
import warnings
from typing import Any, Optional

import torch
from torch import nn

from . import autograd as _autograd
from . import functional as F
from .autograd import matmul_4bit


class Params4bit(torch.nn.Parameter):
    def __new__(cls, data: Optional[torch.Tensor] = None, requires_grad=False, quant_state: Optional[F.QuantState] = None,
                blocksize: int = 64, compress_statistics: bool = True, quant_type: str = "fp4",
                quant_storage: torch.dtype = torch.uint8, module: Optional["Linear4bit"] = None, bnb_quantized: bool = False):
        if data is None:
            data = torch.empty(0)
        self = torch.Tensor._make_subclass(cls, data, requires_grad)
        # NB: the instance __dict__ must hold exactly these constructor kwargs — HF re-creates the
        # parameter as Params4bit(value, requires_grad=False, **old.__dict__).
        self.blocksize = blocksize
        self.compress_statistics = compress_statistics
        self.quant_type = quant_type
        self.quant_state = quant_state
        self.quant_storage = quant_storage
        self.bnb_quantized = bnb_quantized
        self.module = module
        return self

    def __getstate__(self):
        state = self.__dict__.copy()
        state["data"] = self.data
        state["requires_grad"] = self.requires_grad
        return state

    def __setstate__(self, state):
        self.requires_grad = state["requires_grad"]
        self.blocksize = state["blocksize"]
        self.compress_statistics = state["compress_statistics"]
        self.quant_type = state["quant_type"]
        self.quant_state = state["quant_state"]
        self.data = state["data"]
        self.quant_storage = state["quant_storage"]
        self.bnb_quantized = state["bnb_quantized"]
        self.module = state["module"]

    def __deepcopy__(self, memo):
        new = type(self).__new__(type(self))
        state = self.__getstate__()
        new.__setstate__(state)
        new.quant_state = copy.deepcopy(state["quant_state"])
        new.data = copy.deepcopy(state["data"])
        return new

    def __copy__(self):
        new = type(self).__new__(type(self))
        new.__setstate__(self.__getstate__())
        return new

    @classmethod
    def from_prequantized(cls, data: torch.Tensor, quantized_stats: dict[str, Any], requires_grad: bool = False,
                          device="cuda", module: Optional["Linear4bit"] = None, **kwargs) -> "Params4bit":
        self = torch.Tensor._make_subclass(cls, data.to(device))
        self.requires_grad = requires_grad
        self.quant_state = F.QuantState.from_dict(qs_dict=quantized_stats, device=device)
        self.blocksize = self.quant_state.blocksize
        self.compress_statistics = self.quant_state.nested
        self.quant_type = self.quant_state.quant_type
        self.bnb_quantized = True
        self.quant_storage = data.dtype
        self.module = module
        if self.module is not None:
            self.module.quant_state = self.quant_state
        return self

    def _quantize(self, device):
        w = self.data.contiguous().to(device)
        w_4bit, quant_state = F.quantize_4bit(w, blocksize=self.blocksize, compress_statistics=self.compress_statistics,
                                              quant_type=self.quant_type, quant_storage=self.quant_storage)
        self.data = w_4bit
        self.quant_state = quant_state
        if self.module is not None:
            self.module.quant_state = quant_state
        self.bnb_quantized = True
        return self

    def cuda(self, device=None, non_blocking: bool = False):
        return self.to(device="cuda" if device is None else device, non_blocking=non_blocking)

    def cpu(self):
        return self.to(device="cpu")

    def to(self, *args, **kwargs):
        device, dtype, non_blocking, _ = torch._C._nn._parse_to(*args, **kwargs)
        if device is not None and device.type == "cuda" and not self.bnb_quantized:
            # first move to a GPU quantizes (K1 + K2) — qlora.py's from_pretrained(...device_map) path
            return self._quantize(device)
        if self.quant_state is not None and device is not None:
            self.quant_state.to(device)
        # a quantized payload keeps its uint8 storage: dtype casts apply to unquantized data only
        new_data = super().to(device=device, dtype=None if self.bnb_quantized else dtype, non_blocking=non_blocking)
        return Params4bit(new_data, requires_grad=self.requires_grad, quant_state=self.quant_state, blocksize=self.blocksize,
                          compress_statistics=self.compress_statistics, quant_type=self.quant_type,
                          quant_storage=self.quant_storage, module=self.module, bnb_quantized=self.bnb_quantized)


def fix_4bit_weight_quant_state_from_module(module: "Linear4bit"):
    if getattr(module.weight, "quant_state", None) is not None:
        return
    if getattr(module, "quant_state", None) is None:
        warnings.warn("FP4 quantization state not initialized. Please call .cuda() or .to(device) on the LinearFP4 layer first.")
        return
    # the quant state got lost when the parameter got converted (e.g. by FSDP): recover it from the module
    assert module.weight.shape[1] == 1
    if not isinstance(module.weight, Params4bit):
        module.weight = Params4bit(module.weight, quant_storage=module.quant_storage, bnb_quantized=True)
    module.weight.quant_state = module.quant_state


class Linear4bit(nn.Linear):
    """Frozen 4-bit (NF4, optionally double-quantized) linear layer — the QLoRA base layer.

    forward(x): cast x to `compute_dtype`, Y = X . dequant(W)^T (+bias) via the fused kernel,
    cast back to x's dtype (SURVEY.md 8a row a7).  The weight is quantized on first move to CUDA.
    """

    def __init__(self, input_features, output_features, bias=True, compute_dtype=None, compress_statistics=True,
                 quant_type="fp4", quant_storage=torch.uint8, device=None):
        super().__init__(input_features, output_features, bias, device)
        self.weight = Params4bit(self.weight.data, requires_grad=False, compress_statistics=compress_statistics,
                                 quant_type=quant_type, quant_storage=quant_storage, module=self)
        self.compute_dtype = compute_dtype
        self.compute_type_is_set = compute_dtype is not None
        self.quant_state = None
        self.quant_storage = quant_storage

    def set_compute_type(self, x):
        if x.dtype in (torch.float32, torch.bfloat16):
            # the input dtype is safe to compute in: use it
            self.compute_dtype = x.dtype
        elif x.dtype == torch.float16:
            if self.compute_dtype in (None, torch.float32) and x.numel() == x.shape[-1]:
                warnings.warn("Input type into Linear4bit is torch.float16, but bnb_4bit_compute_dtype=torch.float32 (default). This will lead to slow inference.")
                warnings.filterwarnings("ignore", message=".*inference.")
            if self.compute_dtype in (None, torch.float32) and x.numel() != x.shape[-1]:
                warnings.warn("Input type into Linear4bit is torch.float16, but bnb_4bit_compute_dtype=torch.float32 (default). This will lead to slow inference or training speed.")
                warnings.filterwarnings("ignore", message=".*inference or training")

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)  # weight (packed) and bias
        if getattr(self.weight, "quant_state", None) is not None:
            for k, v in self.weight.quant_state.as_dict(packed=True).items():
                destination[prefix + "weight." + k] = v if keep_vars else v.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        # Accept the serialized 4-bit format (keys listed in the module docstring): rebuild the
        # Params4bit from the packed payload + quant-state components, no re-quantization.
        qs_prefix = prefix + "weight."
        qs_keys = [k for k in state_dict if k.startswith(qs_prefix)]
        if qs_keys and (prefix + "weight") in state_dict:
            stats = {k[len(prefix):]: state_dict.pop(k) for k in qs_keys}
            packed = state_dict.pop(prefix + "weight")
            device = packed.device if packed.is_cuda else (self.weight.device if self.weight.is_cuda else "cpu")
            self.weight = Params4bit.from_prequantized(packed, stats, requires_grad=False, device=device, module=self)
            if self.bias is not None and (prefix + "bias") in state_dict:
                with torch.no_grad():
                    self.bias.copy_(state_dict.pop(prefix + "bias"))
            elif self.bias is not None and strict:
                missing_keys.append(prefix + "bias")
            return
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def forward(self, x: torch.Tensor):
        fix_4bit_weight_quant_state_from_module(self)
        # weights are handled by Params4bit, but the bias has to be cast manually
        if self.bias is not None and self.bias.dtype != x.dtype:
            self.bias.data = self.bias.data.to(x.dtype)
        if not self.compute_type_is_set:
            self.set_compute_type(x)
            self.compute_type_is_set = True
        inp_dtype = x.dtype
        if getattr(self.weight, "quant_state", None) is None:
            raise RuntimeError("Linear4bit weight is not quantized yet: move the module to a CUDA device first (.cuda()/.to('cuda'))")
        qs = self.weight.quant_state
        bias = None if self.bias is None else self.bias.to(self.compute_dtype)
        foldable = ((inp_dtype == torch.float32 and self.compute_dtype in (torch.bfloat16, torch.float16))
                    or (inp_dtype == torch.float16 and self.compute_dtype == torch.bfloat16))
        if foldable and x.is_cuda and x.numel() > 0 and _autograd.USE_FUSED and F.fused_supported(qs, self.compute_dtype):
            # fp32 activations (qlora.py:400-401 keeps the norms in fp32; `qlora.py --fp16` loads the whole model in fp32), or
            # fp16 activations under bf16 compute (an fp16 checkpoint loaded with bnb_4bit_compute_dtype=torch.bfloat16):
            # x.to(compute_dtype) and .to(inp_dtype) are folded into the fused node — one input cast, the output cast done by
            # the kernel epilogue (SURVEY.md 8a row a7)
            return matmul_4bit(x, self.weight.t(), bias=bias, quant_state=qs, compute_dtype=self.compute_dtype)
        if self.compute_dtype is not None:
            x = x.to(self.compute_dtype)
        return matmul_4bit(x, self.weight.t(), bias=bias, quant_state=qs).to(inp_dtype)


class LinearNF4(Linear4bit):
    def __init__(self, input_features, output_features, bias=True, compute_dtype=None, compress_statistics=True,
                 quant_storage=torch.uint8, device=None):
        super().__init__(input_features, output_features, bias, compute_dtype, compress_statistics, "nf4", quant_storage, device)


class LinearFP4(Linear4bit):
    def __init__(self, input_features, output_features, bias=True, compute_dtype=None, compress_statistics=True,
                 quant_storage=torch.uint8, device=None):
        super().__init__(input_features, output_features, bias, compute_dtype, compress_statistics, "fp4", quant_storage, device)


class Int8Params(torch.nn.Parameter):
    """Name kept for `bnb.nn.Int8Params` lookups; LLM.int8 is out of scope (north_star is NF4 only)."""

    def __new__(cls, *args, **kwargs):
        raise NotImplementedError("Int8Params / LLM.int8 is outside this build's scope (NF4 Linear4bit only)")


class Linear8bitLt(nn.Linear):
    """Name kept so `qlora.py:249` can evaluate `bnb.nn.Linear8bitLt`; constructing it raises."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("Linear8bitLt / LLM.int8 is outside this build's scope (NF4 Linear4bit only)")
