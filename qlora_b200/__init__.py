"""qlora_b200 — H100-native NF4 + double-quant Linear4bit hot path for QLoRA finetuning.

Drop-in for the slice of `bitsandbytes` that artidoro/qlora uses (qlora.py:15,249,318-326):
`nn.Linear4bit`, `nn.Params4bit`, `matmul_4bit`, `functional.{quantize_4bit, dequantize_4bit,
quantize_blockwise, dequantize_blockwise, QuantState}`.  The hot ops are hand-written sm_90a CUDA
(TMA + in-register NF4 dequant + wgmma) behind the C-ABI in include/qlora_b200.h.
`shims/bitsandbytes` re-exports this package under the import name `bitsandbytes`.
"""
from . import functional, nn, optim  # noqa: F401
from ._lib import LIB_PATH, Qb200Error, is_available  # noqa: F401
from .autograd import MatMul4Bit, matmul_4bit  # noqa: F401
from .lora import LoraMatMul4Bit, lora_linear4bit, lora_linear4bit_group  # noqa: F401
from .lora import DoraMatMul4Bit, dora_linear4bit, dora_linear4bit_group, dora_linear4bit_peft  # noqa: F401
from .mixed import LoraAdapterSet, lora_linear4bit_group_mixed, lora_linear4bit_mixed  # noqa: F401
from .mixed import MultiLoraMatMul4Bit, lora_linear4bit_group_multi, lora_linear4bit_multi  # noqa: F401
from .mixed import DoraAdapterSet, MultiDoraMatMul4Bit, dora_linear4bit_group_multi, dora_linear4bit_multi  # noqa: F401

# transformers gates 4-bit support on `bitsandbytes.__version__ >= 0.46.1`
__version__ = "0.46.1"
supported_torch_devices = {"cuda"}
features = {"multi_backend"}
