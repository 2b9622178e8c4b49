"""CPU tests: the C-ABI library loads and exports every symbol include/qlora_b200.h declares (no
compute without a GPU), and the Python host mirrors the bitsandbytes surface the reference binds."""
import copy
import os
import pickle
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "qlora_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(?:int64_t|int|void|const char\*)\s+\**\s*([a-z][a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import ctypes as ct

    from qlora_b200 import _build, _lib

    _build.build()
    lib = ct.CDLL(_lib.LIB_PATH)
    names = _header_functions()
    assert len(names) >= 18 and "qb200_nf4_linear_fwd" in names and "cdequantize_blockwise_bf16_nf4" in names
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/qlora_b200.h but not exported"
    assert set(_lib.EXPORTED_SYMBOLS) == set(names)
    lib.qb200_last_error.restype = ct.c_char_p
    assert lib.qb200_version() == 100 and lib.qb200_has_fused_gemm() == 1
    assert lib.qb200_last_error() == b""


def test_argument_errors_do_not_need_a_gpu():
    """Validation happens before any launch: bad arguments return QB200_E* with a message."""
    from qlora_b200 import _lib

    lib = _lib.load()
    assert lib.qb200_quantize_nf4(None, 2, 64, 64, None, None, None) == -1
    assert b"null pointer" in lib.qb200_last_error()
    buf = (__import__("ctypes").c_char * 256)()
    p = __import__("ctypes").cast(buf, __import__("ctypes").c_void_p)
    assert lib.qb200_quantize_nf4(p, 7, 64, 64, p, p, None) == -1
    assert lib.qb200_quantize_nf4(p, 2, 64, 100, p, p, None) == -1
    assert b"blocksize" in lib.qb200_last_error()
    # fused GEMM shape checks
    assert lib.qb200_nf4_linear_fwd(p, p, None, None, None, None, p, None, p, 8, 128, 96, None) == -2  # K % 64
    assert b"multiple of 64" in lib.qb200_last_error()
    assert lib.qb200_nf4_linear_fwd(p, p, None, None, None, None, None, None, p, 8, 128, 128, None) == -1  # no absmax


def test_sass_is_hopper_native():
    """The shipped .so must contain sm_90a warpgroup-MMA and TMA SASS (HGMMA, UTMALDG)."""
    from qlora_b200 import _lib

    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG"):
        assert mnemonic in sass, mnemonic
    # warp-level mma.sync (HMMA) is allowed in exactly one place: the <= 32-token skinny forward kernel, which is bound by the
    # NF4 look-up on the ALU pipe and feeds the look-up registers straight into the MMA (DESIGN.md); every GEMM-sized
    # launch is wgmma (HGMMA)
    fn = None
    for line in sass.splitlines():
        if "Function :" in line:
            fn = line
        elif "HMMA." in line:
            assert fn is not None and "nf4_skinny_kernel" in fn, fn


def test_cpu_tensors_fail_loudly():
    import qlora_b200 as q

    with pytest.raises(RuntimeError, match="CUDA"):
        q.functional.quantize_4bit(torch.randn(128), quant_type="nf4")
    lin = q.nn.Linear4bit(64, 64, bias=False, compute_dtype=torch.bfloat16, quant_type="nf4")
    with pytest.raises(RuntimeError):
        lin(torch.randn(2, 64))  # not quantized / not on CUDA: no silent CPU path


def test_surface_matches_reference_touch_points():
    """qlora.py:15,249 — type identity through the shim; find_all_linear_names' logic (qlora.py:248-259)."""
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    import bitsandbytes as bnb
    import qlora_b200 as q

    assert bnb.nn.Linear4bit is q.nn.Linear4bit and bnb.nn.Params4bit is q.nn.Params4bit
    assert issubclass(bnb.nn.Linear4bit, torch.nn.Linear) and issubclass(bnb.nn.Linear8bitLt, torch.nn.Linear)
    assert tuple(int(x) for x in bnb.__version__.split(".")) >= (0, 46, 1) and "cuda" in bnb.supported_torch_devices
    from bitsandbytes.functional import QuantState, dequantize_4bit, quantize_4bit  # noqa: F401
    import bitsandbytes.nn.modules as m  # noqa: F401

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj = bnb.nn.Linear4bit(64, 64, bias=False, compute_dtype=torch.bfloat16, compress_statistics=True, quant_type="nf4")
            self.up_proj = bnb.nn.LinearNF4(64, 128, bias=False)
            self.norm = torch.nn.LayerNorm(64)
            self.lm_head = torch.nn.Linear(64, 10)

    model = Block()
    cls = bnb.nn.Linear4bit
    names = set()
    for name, module in model.named_modules():
        if isinstance(module, cls):
            parts = name.split(".")
            names.add(parts[0] if len(parts) == 1 else parts[-1])
    assert names == {"q_proj", "up_proj"}
    with pytest.raises(NotImplementedError):
        bnb.nn.Linear8bitLt(4, 4)


def test_params4bit_contract():
    import qlora_b200 as q

    w = torch.randn(32, 64)
    p = q.nn.Params4bit(w, requires_grad=False, compress_statistics=True, quant_type="nf4")
    # HF re-creates the parameter from __dict__ (transformers/integrations/bitsandbytes.py:85-91)
    assert set(p.__dict__) == {"blocksize", "compress_statistics", "quant_type", "quant_state", "quant_storage", "bnb_quantized", "module"}
    p2 = q.nn.Params4bit(w.clone(), requires_grad=False, **p.__dict__)
    assert p2.quant_type == "nf4" and p2.blocksize == 64 and not p2.bnb_quantized and not p2.requires_grad
    assert isinstance(p, torch.nn.Parameter)
    p3 = copy.deepcopy(p)
    assert torch.equal(p3.data, p.data) and p3.quant_type == "nf4"
    p4 = pickle.loads(pickle.dumps(p))
    assert torch.equal(p4.data, p.data) and p4.compress_statistics
    # moving between CPU dtypes/devices does not quantize; only the first move to CUDA does
    assert not p.to("cpu").bnb_quantized
    lin = q.nn.Linear4bit(64, 32, bias=True, compute_dtype=torch.bfloat16, compress_statistics=False, quant_type="nf4")
    assert lin.compute_dtype == torch.bfloat16 and lin.weight.module is lin and not lin.weight.compress_statistics
    assert lin.in_features == 64 and lin.out_features == 32 and lin.weight.quant_type == "nf4"


def test_quant_state_dict_roundtrip_cpu():
    from qlora_b200.functional import QuantState, create_dynamic_map, get_4bit_type

    code = create_dynamic_map()
    st2 = QuantState(absmax=torch.rand(2), code=code, blocksize=256, dtype=torch.float32)
    qs = QuantState(absmax=torch.randint(0, 255, (384,), dtype=torch.uint8), shape=torch.Size([96, 256]), dtype=torch.bfloat16,
                    blocksize=64, quant_type="nf4", code=get_4bit_type("nf4", device="cpu"), offset=torch.tensor(0.0521), state2=st2)
    assert qs.nested and qs[0] is qs.absmax and qs[4][1] is st2 and qs[5] == "nf4"  # list-style (0.40-era) access
    packed = qs.as_dict(packed=True)
    assert set(packed) == {"absmax", "quant_map", "nested_absmax", "nested_quant_map", "quant_state.bitsandbytes__nf4"}
    assert all(isinstance(v, torch.Tensor) for v in packed.values())
    back = QuantState.from_dict({"weight." + k: v for k, v in packed.items()}, device="cpu")
    assert back.shape == qs.shape and back.dtype == torch.bfloat16 and back.blocksize == 64 and back.nested
    assert torch.equal(back.absmax, qs.absmax) and torch.equal(back.state2.absmax, st2.absmax)
    assert abs(back.offset.item() - 0.0521) < 1e-7 and back.state2.blocksize == 256
    with pytest.raises(ValueError):
        QuantState.from_dict({"foo": 1}, device="cpu")


def test_dynamic_map_equals_oracle():
    from oracle import nf4_oracle as o
    from qlora_b200.functional import create_dynamic_map, create_normal_map, get_4bit_type
    import numpy as np

    assert np.array_equal(create_dynamic_map().numpy(), o.create_dynamic_map())
    assert np.array_equal(get_4bit_type("nf4", device="cpu").numpy(), o.NF4_LUT)
    assert np.array_equal(create_normal_map()[:16].numpy(), o.NF4_LUT)


def test_product_does_not_import_oracle():
    """The shipped package must never route through the oracle (test infrastructure)."""
    pkg = os.path.join(ROOT, "qlora_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "nf4_oracle" not in text, f


def test_optim_surface():
    """qlora.py:198 optim='paged_adamw_32bit' -> HF builds bitsandbytes.optim.AdamW(is_paged=True, optim_bits=32)."""
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    import bitsandbytes as bnb
    from bitsandbytes.optim import AdamW, GlobalOptimManager, PagedAdamW32bit

    p = torch.nn.Parameter(torch.zeros(8))
    opt = AdamW([p], lr=2e-4, betas=(0.9, 0.999), eps=1e-8, optim_bits=32, is_paged=True)
    assert opt.is_paged and isinstance(opt, torch.optim.Optimizer) and issubclass(PagedAdamW32bit, AdamW)
    with pytest.raises(NotImplementedError):
        AdamW([p], optim_bits=8)
    p.grad = torch.ones(8)
    with pytest.raises(RuntimeError, match="CUDA"):
        opt.step()   # CPU parameter: no CPU fallback
    assert GlobalOptimManager.get_instance() is GlobalOptimManager.get_instance()
    assert bnb.optim.PagedAdamW is not None


def test_device_constants_match_oracle():
    """The numeric constants compiled into the CUDA path (no GPU needed to read them): the NF4 codebook and the 33-cell
    classification table of K1 (`QB200_NF4_CELLS_INIT`, nf4_common.cuh) reproduce the oracle's codebook / threshold tree.
    The table is emulated exactly as the kernel evaluates it: cell = low bits of fl(16 x + (2^23 + 16)),
    code = base[cell] + (x > thr[cell]), NaN -> cell 0."""
    import re

    import numpy as np

    from oracle import nf4_oracle as o

    src = open(os.path.join(ROOT, "qlora_b200", "csrc", "nf4_common.cuh")).read()
    lut_txt = src[src.index("#define QB200_NF4_LUT_INIT"):src.index("// A.2")]
    lut = np.array([float(v.rstrip("f")) for v in re.findall(r"-?\d+\.\d+f", lut_txt)], dtype=np.float32)
    assert np.array_equal(lut, o.NF4_LUT.astype(np.float32))
    cells_txt = src[src.index("#define QB200_NF4_CELLS_INIT"):src.index("constexpr int kNf4Cells")]
    cells = re.findall(r"\{0x([0-9a-f]{8})u, (\d+)u\}", cells_txt)
    assert len(cells) == 33
    thr = np.array([int(h, 16) for h, _ in cells], dtype=np.uint32).view(np.float32)
    base = np.array([int(b) for _, b in cells], dtype=np.uint32)
    # every oracle threshold appears exactly once, in ascending order, and base counts the thresholds in lower cells
    finite = thr[np.isfinite(thr)]
    assert np.array_equal(finite, o.NF4_THRESHOLDS.astype(np.float32))
    assert np.array_equal(base, np.concatenate([[0], np.cumsum(np.isfinite(thr))[:-1]]).astype(np.uint32))

    def code_cells(x):
        xc = np.minimum(np.maximum(np.where(np.isnan(x), np.float32(-1.0), x), np.float32(-1.0)), np.float32(1.0))
        t = (xc * np.float32(16.0)).astype(np.float32) + np.float32(8388624.0)       # 16 x is exact: the add rounds like the fma
        cell = (t.astype(np.float32).view(np.uint32) - np.uint32(0x4B000000)).astype(np.int64)
        assert cell.min() >= 0 and cell.max() <= 32
        return (base[cell] + (xc > thr[cell])).astype(np.uint8)

    rng = np.random.default_rng(7)
    xs = [rng.uniform(-1, 1, 2_000_000).astype(np.float32)]
    centres = list(o.NF4_THRESHOLDS.astype(np.float32)) + [np.float32(k / 16.0 - 1.0 + d) for k in range(33) for d in (0.0, 1.0 / 32)]
    for c in centres:
        bits = np.float32(c).view(np.uint32).astype(np.int64) + np.arange(-2000, 2001)
        nb = bits.astype(np.uint32).view(np.float32)
        xs.append(nb[np.abs(nb) <= np.float32(1.0000001)])
    xs.append(np.array([np.nan, 0.0, -0.0, 1.0, -1.0, np.nextafter(np.float32(1), np.float32(2))], dtype=np.float32))
    x = np.concatenate(xs)
    assert np.array_equal(code_cells(x), o.quantize_nf4_codes(x))
