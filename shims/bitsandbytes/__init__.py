"""Import-name shim: `import bitsandbytes as bnb` resolves to qlora_b200.

Put `<repo>/shims` on PYTHONPATH (see INTEGRATION.md) and the reference's three touch-points
(qlora.py:15 import, qlora.py:249 `bnb.nn.Linear4bit`/`bnb.nn.Linear8bitLt`, qlora.py:318-326
BitsAndBytesConfig -> HF -> `bnb.nn.Linear4bit(...)`, `bnb.nn.Params4bit(...)`) bind to the H100 path.
"""
import os as _os
import sys as _sys

_root = _os.path.dirname(_os.path.dirname(_os.path.dirname(_os.path.abspath(__file__))))
if _root not in _sys.path:
    _sys.path.insert(0, _root)

import qlora_b200 as _impl  # noqa: E402
from qlora_b200 import MatMul4Bit, matmul_4bit  # noqa: E402,F401
from qlora_b200 import lora_linear4bit, lora_linear4bit_group  # noqa: E402,F401  (extensions: fused LoRA step, SURVEY.md 8f-1)
from qlora_b200 import dora_linear4bit, dora_linear4bit_group, dora_linear4bit_peft  # noqa: E402,F401  (extensions: fused QDoRA)
# extensions: mixed-adapter batches (peft adapter_names)
from qlora_b200 import LoraAdapterSet, lora_linear4bit_group_mixed, lora_linear4bit_mixed  # noqa: E402,F401
# extensions: several adapters trained over one base in one batch
from qlora_b200 import lora_linear4bit_group_multi, lora_linear4bit_multi  # noqa: E402,F401
from qlora_b200 import DoraAdapterSet, dora_linear4bit_group_multi, dora_linear4bit_multi  # noqa: E402,F401
from qlora_b200 import functional, nn, optim  # noqa: E402,F401

__version__ = _impl.__version__
supported_torch_devices = _impl.supported_torch_devices
features = _impl.features

# `import bitsandbytes.nn`, `from bitsandbytes.functional import ...`, `bitsandbytes.nn.modules` (peft)
_sys.modules[__name__ + ".functional"] = functional
_sys.modules[__name__ + ".nn"] = nn
_sys.modules[__name__ + ".nn.modules"] = nn
nn.modules = nn  # `import bitsandbytes.nn.modules as m` resolves by attribute
_sys.modules[__name__ + ".optim"] = optim
_sys.modules[__name__ + ".autograd"] = _impl.autograd
_sys.modules[__name__ + ".autograd._functions"] = _impl.autograd


