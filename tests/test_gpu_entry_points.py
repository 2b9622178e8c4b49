"""The public NF4 linear entry points agree with one another: each gives bitwise the output of `functional.nf4_linear_group`
for the same problem.  That covers the five single-problem forms (`qb200_nf4_linear_fwd`, `_bwd_dx`, `_fwd_lora`,
`_bwd_dx_lora`, `_ex`) and the four grouped ones (`qb200_nf4_linear_group`, `_scaled`, `_typed`, `_ex`).

Split-K changes the summation order, so an entry point that takes a workspace gets one large enough for both the split-K
partials and the bf16 weight scratch, as `nf4_linear_group` allocates.  The four forms without a workspace run the fused
kernel unsplit: below the scratch threshold they are compared with `qb200_nf4_linear_group` given no workspace, at training
token counts with `nf4_linear_group` (the fused and scratch paths are bitwise equal there).  M = 1, 8, 300 and 2048 reach the
skinny, fused (split-K included) and scratch paths."""
import ctypes as ct
import functools

import pytest
import torch

from gpu_helpers import make_act, make_weight

BF16, H16, F32 = torch.bfloat16, torch.float16, torch.float32
N, K, R = 512, 1024, 16
MS = [1, 8, 300, 2048]
# (is_bwd, LoRA operands, bias)
DIRECTIONS = [(False, False, False), (False, False, True), (False, True, True), (True, False, False), (True, True, False)]


@pytest.fixture(scope="module")
def F():
    import qlora_b200.functional as F

    return F


def _lib():
    from qlora_b200 import _lib

    return _lib.load()


def _code(dt):
    from qlora_b200._lib import DTYPE_CODE

    return DTYPE_CODE[dt]


@functools.lru_cache(maxsize=None)
def _quant(nested, state_dtype):
    import qlora_b200.functional as F

    packed, qs = F.quantize_4bit(make_weight(N, K, seed=3, dtype=state_dtype), compress_statistics=nested, quant_type="nf4")
    return packed.contiguous(), qs


def _operands(is_bwd, lora, bias, m, cdt, seed=1):
    x = make_act(m, N if is_bwd else K, seed).to(cdt)
    u = make_act(m, R, seed + 1).to(cdt) if lora else None
    v = (make_weight(R, K, seed + 2) if is_bwd else make_weight(N, R, seed + 2)).to(cdt) if lora else None
    b = make_weight(1, N, seed + 3)[0].to(cdt) if bias else None
    return x, u, v, b


def _ptr(t):
    return None if t is None else t.data_ptr()


def _state_ptrs(qs):
    """(absmax_u8, code256, absmax2, offset, absmax_f32) as the kernels read them."""
    if qs.nested:
        return _ptr(qs.absmax), _ptr(qs.state2.code), _ptr(qs.state2.absmax), _ptr(qs.offset), None
    return None, None, None, None, _ptr(qs.absmax)


class _Case:
    """One problem: its operands, the reference output of `nf4_linear_group`, and a caller for each C entry point."""

    def __init__(self, F, is_bwd, lora, bias, m, cdt, nested=True, state_dtype=BF16, out_dtype=None, row_scale=False):
        self.F, self.lib = F, _lib()
        self.is_bwd, self.m, self.cdt = is_bwd, m, cdt
        self.out_dtype = cdt if out_dtype is None else out_dtype
        self.packed, self.qs = _quant(nested, state_dtype)
        self.x, self.u, self.v, self.b = _operands(is_bwd, lora, bias, m, cdt)
        self.r = R if lora else 0
        self.scale = (torch.rand(N, generator=torch.Generator().manual_seed(9)) + 0.5).cuda() if row_scale else None
        self.f_out = K if is_bwd else N
        ws = max(self.lib.qb200_nf4_linear_workspace_size(m, N, K, int(is_bwd)),
                 self.lib.qb200_nf4_linear_scratch_size(1, m, N, K, int(is_bwd)))
        self.ws = torch.empty(ws, dtype=torch.uint8, device="cuda") if ws else None
        self.ws_bytes = ws
        self.stream = F.stream_ptr(self.x.device)
        ref = F.nf4_linear_group(is_bwd, [self.x], [self.packed], [self.qs], None if self.b is None else [self.b],
                                 None if self.u is None else [self.u], None if self.v is None else [self.v],
                                 out_dtype=self.out_dtype, row_scales=None if self.scale is None else [self.scale])
        self.ref = ref if is_bwd else ref[0]

    def _out(self):
        return torch.full((self.m, self.f_out), float("nan"), dtype=self.out_dtype, device="cuda")

    def _check(self, rc, out, ref, what):
        assert rc == 0, (what, rc, self.lib.qb200_last_error())
        torch.cuda.synchronize()
        assert torch.equal(out, ref), what

    def _problems(self, out):
        from qlora_b200._lib import Nf4Problem

        a_u8, code, a2, off, a32 = _state_ptrs(self.qs)
        pr = Nf4Problem(inp=_ptr(self.x), packed=_ptr(self.packed), absmax_u8=a_u8, code256=code, absmax2=a2, offset=off,
                        absmax_f32=a32, bias=_ptr(self.b), U=_ptr(self.u), V=_ptr(self.v), out=_ptr(out))
        return (Nf4Problem * 1)(pr)

    def _run_group(self, name, lead, ws):
        out = self._out()
        probs = self._problems(out)
        args = [int(self.is_bwd), *lead, 1, ct.addressof(probs)]
        if name in ("qb200_nf4_linear_group_scaled", "qb200_nf4_linear_group_typed"):
            scales = (ct.c_void_p * 1)(_ptr(self.scale))
            args.append(None if self.scale is None else ct.addressof(scales))
        args += [self.r, self.m, N, K, _code(self.out_dtype), _ptr(self.ws) if ws else None, self.ws_bytes if ws else 0, self.stream]
        return getattr(self.lib, name)(*args), out

    def group(self, name, *lead):
        """A grouped entry point: `lead` are its arguments between is_bwd and nprob."""
        rc, out = self._run_group(name, lead, ws=True)
        self._check(rc, out, self.ref, name)

    def single(self, name):
        """A single-problem entry point (bf16 throughout)."""
        out = self._out()
        state = (_ptr(self.x), _ptr(self.packed), *_state_ptrs(self.qs))
        if name == "qb200_nf4_linear_ex":
            rc = self.lib.qb200_nf4_linear_ex(int(self.is_bwd), *state, _ptr(self.b), _ptr(self.u), _ptr(self.v), self.r, _ptr(out),
                                              self.m, N, K, _ptr(self.ws), self.ws_bytes, self.stream)
            self._check(rc, out, self.ref, name)
            return
        if name == "qb200_nf4_linear_fwd":
            rc = self.lib.qb200_nf4_linear_fwd(*state, _ptr(self.b), _ptr(out), self.m, N, K, self.stream)
        elif name == "qb200_nf4_linear_bwd_dx":
            rc = self.lib.qb200_nf4_linear_bwd_dx(*state, _ptr(out), self.m, N, K, self.stream)
        elif name == "qb200_nf4_linear_fwd_lora":
            rc = self.lib.qb200_nf4_linear_fwd_lora(*state, _ptr(self.b), _ptr(self.u), _ptr(self.v), self.r, _ptr(out), self.m, N, K,
                                                    self.stream)
        else:
            rc = self.lib.qb200_nf4_linear_bwd_dx_lora(*state, _ptr(self.u), _ptr(self.v), self.r, _ptr(out), self.m, N, K, self.stream)
        # no workspace: the fused kernel, unsplit, at every token count
        ref = self.ref
        if self.lib.qb200_nf4_linear_scratch_size(1, self.m, N, K, int(self.is_bwd)) == 0:
            rc_ref, ref = self._run_group("qb200_nf4_linear_group", (), ws=False)
            assert rc_ref == 0, self.lib.qb200_last_error()
        self._check(rc, out, ref, name)


@pytest.mark.gpu
@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("is_bwd,lora,bias", DIRECTIONS)
@pytest.mark.parametrize("nested,state_dtype", [(True, BF16), (False, BF16), (True, F32)])
def test_bf16_entry_points_match_nf4_linear_group(F, m, is_bwd, lora, bias, nested, state_dtype):
    c = _Case(F, is_bwd, lora, bias, m, BF16, nested, state_dtype)
    c.single("qb200_nf4_linear_ex")
    c.group("qb200_nf4_linear_group")
    c.group("qb200_nf4_linear_group_typed", _code(BF16))
    c.group("qb200_nf4_linear_group_ex", _code(BF16), _code(state_dtype))
    c.single(("qb200_nf4_linear_bwd_dx" if is_bwd else "qb200_nf4_linear_fwd") + ("_lora" if lora else ""))
    # an fp32 output: the bf16-rounded result widened in the epilogue
    c = _Case(F, is_bwd, lora, bias, m, BF16, nested, state_dtype, out_dtype=F32)
    c.group("qb200_nf4_linear_group")
    c.group("qb200_nf4_linear_group_typed", _code(BF16))
    c.group("qb200_nf4_linear_group_ex", _code(BF16), _code(state_dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("is_bwd,lora,bias", DIRECTIONS)
@pytest.mark.parametrize("state_dtype", [H16, F32])
@pytest.mark.parametrize("out_dtype", [H16, F32])
def test_fp16_compute_entry_points_match_nf4_linear_group(F, m, is_bwd, lora, bias, state_dtype, out_dtype):
    c = _Case(F, is_bwd, lora, bias, m, H16, state_dtype=state_dtype, out_dtype=out_dtype)
    c.group("qb200_nf4_linear_group_typed", _code(H16))
    c.group("qb200_nf4_linear_group_ex", _code(H16), _code(state_dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("is_bwd,lora,bias", DIRECTIONS)
@pytest.mark.parametrize("out_dtype", [H16, BF16])
def test_fp16_state_under_bf16_compute_matches_nf4_linear_group(F, m, is_bwd, lora, bias, out_dtype):
    c = _Case(F, is_bwd, lora, bias, m, BF16, state_dtype=H16, out_dtype=out_dtype)
    c.group("qb200_nf4_linear_group_ex", _code(BF16), _code(H16))


@pytest.mark.gpu
@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("is_bwd,lora,bias", DIRECTIONS)
@pytest.mark.parametrize("cdt", [BF16, H16])
def test_row_scaled_entry_points_match_nf4_linear_group(F, m, is_bwd, lora, bias, cdt):
    c = _Case(F, is_bwd, lora, bias, m, cdt, state_dtype=cdt, row_scale=True)
    if cdt == BF16:
        c.group("qb200_nf4_linear_group_scaled")
    c.group("qb200_nf4_linear_group_typed", _code(cdt))
