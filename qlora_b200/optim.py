"""`bitsandbytes.optim` surface for the optimizer QLoRA uses: 32-bit AdamW, optionally with *paged* state.

Reference touch-point: qlora.py:198 `optim='paged_adamw_32bit'` -> HF `Trainer` builds
`bitsandbytes.optim.AdamW(params, lr=..., betas=..., eps=..., optim_bits=32, is_paged=True)`
[transformers/trainer_optimizer.py].  Upstream keeps the fp32 moments in CUDA unified memory so that they can be
evicted to host RAM under memory pressure (`cget_managed_ptr`, `cprefetch`) and updates with one fused kernel
(`kOptimizer32bit2State`).  Same here (SURVEY.md 8f-3): `qb200_managed_alloc` / `qb200_prefetch` /
`qb200_adamw32bit_step` behind the C-ABI; the update touches only the trainable (LoRA) parameters.
The Trainer's other 32-bit bitsandbytes names build `Lion`, `RMSprop` and `AdEMAMix` (one kernel, csrc/optim32.cu),
which share AdamW's plumbing through `_Optimizer32bit`.
Only the 32-bit variants exist; 8-bit optimizers raise NotImplementedError.
"""
from __future__ import annotations

import ctypes as ct

import torch

from . import _lib
from ._lib import DTYPE_CODE, check, ptr, stream_ptr


class _ManagedBuffer:
    """fp32 buffer in CUDA unified memory, exposed to torch through __cuda_array_interface__."""

    def __init__(self, numel: int, device: torch.device):
        self.numel = numel
        self.nbytes = 4 * numel
        self.device = device
        out = ct.c_void_p()
        with torch.cuda.device(device):
            check(_lib.load().qb200_managed_alloc(self.nbytes, ct.byref(out)), "managed_alloc")
        self.ptr = out.value
        self.__cuda_array_interface__ = {"shape": (numel,), "typestr": "<f4", "data": (self.ptr, False), "version": 2}
        self.tensor = torch.as_tensor(self, device=device)
        self.tensor.zero_()

    def prefetch(self, to_device: bool = True):
        dev = self.device.index if to_device else -1
        check(_lib.load().qb200_prefetch(ct.c_void_p(self.ptr), self.nbytes, dev, stream_ptr(self.device)), "prefetch")

    def __del__(self):
        try:
            if getattr(self, "ptr", None):
                self.tensor = None
                _lib.load().qb200_managed_free(ct.c_void_p(self.ptr))
                self.ptr = None
        except Exception:
            pass


class _Optimizer32bit(torch.optim.Optimizer):
    """Plumbing shared by the 32-bit optimizers; a subclass names its fp32 state buffers and its launch.

    `self.state[p]` holds tensors only (`step`, `state1`, ...), as upstream's does: the unified-memory allocations that back
    paged state live in `self._paged` (never pickled), and `load_state_dict` re-homes loaded state into freshly allocated
    managed buffers — `optimizer.pt` written by HF Trainer therefore carries no raw device pointers.

    `capturable=True` (extension): the step count lives in one device scalar and the update reads it (and an optional
    device-side gradient scale, `step(grad_scale=...)`) from device memory, so `step()` can be captured in a CUDA graph.
    """

    _NAME = ""
    _STATE_ROWS: tuple = ()   # rows of state1, state2, ...: 1 -> [numel], k > 1 -> [k, numel] (k stacked buffers)
    _READS_STEP = True        # the launch reads the step count (eager steps write each parameter's count to the device first)

    def __init__(self, params, defaults, is_paged, capturable):
        self.is_paged = is_paged
        self.capturable = capturable
        self._paged: dict = {}       # id(param) -> tuple of _ManagedBuffer; owners of the unified memory
        self._step_dev = None        # capturable: device float32 scalar, shared by every parameter
        self._step_eager = None      # not capturable: device copy of the count of the parameter being updated
        self._flat = None            # step_flat: the state buffers over the whole flat parameter buffer
        self._flat_offsets = None    # step_flat: offset of every parameter (param_groups order) in the flat buffer
        super().__init__(params, defaults)

    def _state_keys(self):
        return tuple(f"state{i + 1}" for i in range(len(self._STATE_ROWS)))

    def _new_moments(self, p):
        n = p.numel()
        if self.is_paged:
            bufs = tuple(_ManagedBuffer(rows * n, p.device) for rows in self._STATE_ROWS)
            self._paged[id(p)] = bufs
            flat = [b.tensor for b in bufs]
        else:
            flat = [torch.zeros(rows * n, dtype=torch.float32, device=p.device) for rows in self._STATE_ROWS]
        return tuple(t if rows == 1 else t.view(rows, n) for t, rows in zip(flat, self._STATE_ROWS))

    def _init_state(self, p):
        st = self.state[p]
        st["step"] = torch.zeros((), dtype=torch.float32)   # host tensor, like torch.optim (capturable: see _step_dev)
        st.update(zip(self._state_keys(), self._new_moments(p)))

    def _launch(self, p, g, states, group, step_dev, grad_scale):
        """One update of `p` (any CUDA tensor: a parameter or the flat buffer) from `g` with the step count at `step_dev`."""
        raise NotImplementedError

    def _launch_eager(self, p, g, states, group, step: int):
        step_dev = None
        if self._READS_STEP:
            if self._step_eager is None or self._step_eager.device != p.device:
                self._step_eager = torch.zeros((), dtype=torch.float32, device=p.device)
            self._step_eager.fill_(float(step))
            step_dev = self._step_eager
        self._launch(p, g, states, group, step_dev, None)

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        # torch's loader casts floating-point state to the PARAMETER's dtype (bf16 adapters would get bf16 moments): take the
        # fp32 state from the file itself.  Paged optimizers give it fresh unified-memory homes; a pointer is never adopted
        # from the file.
        self._paged.clear()
        self._flat = None   # a later step_flat rebuilds its flat state from the loaded per-parameter slices
        saved_groups = state_dict["param_groups"]
        id_to_param = {}
        for g_saved, g in zip(saved_groups, self.param_groups):
            for pid, p in zip(g_saved["params"], g["params"]):
                id_to_param[pid] = p
        last = 0.0
        for pid, st_saved in state_dict["state"].items():
            p = id_to_param[pid]
            st = self.state[p]
            loaded = [torch.as_tensor(st_saved[k]).detach().to(device=p.device, dtype=torch.float32) for k in self._state_keys()]
            for k, t, src in zip(self._state_keys(), self._new_moments(p), loaded):
                t.copy_(src.reshape(t.shape))
                st[k] = t
            step = st_saved.get("step", 0)
            st["step"] = torch.tensor(float(step), dtype=torch.float32)
            last = max(last, float(st["step"]))
        if self.capturable:
            if self._step_dev is None and id_to_param:
                dev = next(iter(id_to_param.values())).device
                self._step_dev = torch.zeros((), dtype=torch.float32, device=dev)
            if self._step_dev is not None:
                self._step_dev.fill_(last)

    @torch.no_grad()
    def step(self, closure=None, grad_scale: torch.Tensor | None = None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        bumped = False
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda:
                    raise RuntimeError(f"qlora_b200.optim.{self._NAME} updates CUDA parameters only (no CPU fallback)")
                if p.dtype not in DTYPE_CODE or p.grad.dtype != p.dtype:
                    raise ValueError(f"unsupported parameter/gradient dtype {p.dtype}/{p.grad.dtype}")
                if p.grad.is_sparse:
                    raise RuntimeError("sparse gradients are not supported")
                if not p.is_contiguous():
                    raise RuntimeError("parameters must be contiguous")
                st = self.state[p]
                if len(st) == 0:
                    self._init_state(p)
                if self.is_paged and id(p) in self._paged and not torch.cuda.is_current_stream_capturing():
                    for b in self._paged[id(p)]:
                        b.prefetch(True)
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                states = tuple(st[k] for k in self._state_keys())
                with torch.cuda.device(p.device):
                    if self.capturable:
                        if self._step_dev is None:
                            self._step_dev = torch.zeros((), dtype=torch.float32, device=p.device)
                        if not bumped:   # one device-side increment per step() call (captured with the rest)
                            self._step_dev.add_(1.0)
                            bumped = True
                        self._launch(p, g, states, group, self._step_dev, grad_scale)
                    else:
                        if grad_scale is not None:
                            raise ValueError("grad_scale needs capturable=True (device-side scalars)")
                        st["step"] += 1
                        self._launch_eager(p, g, states, group, int(st["step"]))
        return loss

    @torch.no_grad()
    def step_flat(self, flat_param: torch.Tensor, flat_grad: torch.Tensor, grad_scale: torch.Tensor | None = None):
        """ONE launch for ALL parameters when they (and their gradients) are views into two flat buffers of identical layout
        (harness/dp.py keeps the LoRA adapters that way): `flat_param[i]` is updated from `flat_grad[i]` with one set of
        flat fp32 state buffers (paged when `is_paged`).  Needs `capturable=True`; every parameter of the optimizer must be a
        view into `flat_param` and share one hyper-parameter group.  `state_dict()` publishes the flat state as per-parameter
        `state1` / `state2` slices; state loaded by `load_state_dict` is copied into the flat buffers by the next call."""
        if not self.capturable:
            raise ValueError("step_flat needs capturable=True")
        if len(self.param_groups) != 1:
            raise ValueError("step_flat supports a single parameter group")
        group = self.param_groups[0]
        if flat_param.dtype not in DTYPE_CODE or flat_grad.dtype != flat_param.dtype or flat_param.numel() != flat_grad.numel():
            raise ValueError("flat parameter / gradient buffers must share dtype and size")
        if not (flat_param.is_cuda and flat_param.is_contiguous() and flat_grad.is_contiguous()):
            raise RuntimeError("flat buffers must be contiguous CUDA tensors")
        total = sum(p.numel() for p in group["params"])
        if total != flat_param.numel():
            raise ValueError("the flat buffer does not cover exactly the optimizer's parameters")
        if self._flat is None:
            self._flat_offsets = self._offsets_in(flat_param, group["params"])
            class _P:   # stand-in carrying numel / device for _new_moments
                pass
            proxy = _P()
            proxy.numel = flat_param.numel
            proxy.device = flat_param.device
            self._flat_key = proxy
            bufs = self._new_moments(proxy)
            for p, off in zip(group["params"], self._flat_offsets):   # state from load_state_dict (or per-parameter steps)
                st = self.state.pop(p, None)
                if st and "state1" in st:
                    for k, b in zip(self._state_keys(), bufs):
                        dst = b[..., off:off + p.numel()]
                        dst.copy_(st[k].reshape(dst.shape))
                self._paged.pop(id(p), None)
            self._flat = bufs
        with torch.cuda.device(flat_param.device):
            if self._step_dev is None:
                self._step_dev = torch.zeros((), dtype=torch.float32, device=flat_param.device)
            self._step_dev.add_(1.0)
            if self.is_paged and not torch.cuda.is_current_stream_capturing():
                for b in self._paged.get(id(self._flat_key), ()):
                    b.prefetch(True)
            self._launch(flat_param, flat_grad, self._flat, group, self._step_dev, grad_scale)

    @staticmethod
    def _offsets_in(flat: torch.Tensor, params) -> list:
        """Element offset of every parameter in `flat`; each must be a contiguous view into it, and together they cover it."""
        offs, base, es = [], flat.data_ptr(), flat.element_size()
        for p in params:
            off, rem = divmod(p.data_ptr() - base, es)
            if rem or off < 0 or off + p.numel() > flat.numel() or not p.is_contiguous() or p.dtype != flat.dtype:
                raise ValueError("step_flat: every parameter must be a contiguous view into the flat parameter buffer")
            offs.append(off)
        end = 0
        for off, n in sorted(zip(offs, (p.numel() for p in params))):
            if off != end:
                raise ValueError("step_flat: the parameters overlap or leave a gap in the flat parameter buffer")
            end = off + n
        return offs

    def state_dict(self):
        t = None
        if self.capturable and self._step_dev is not None:   # publish the device-side count in the per-parameter `step`s
            t = float(self._step_dev.item())
            for st in self.state.values():
                if "step" in st:
                    st["step"] = torch.tensor(t, dtype=torch.float32)
        sd = super().state_dict()
        if self._flat is not None:   # step_flat's state, one slice per parameter (views: torch.save writes the buffer once)
            for i, (p, off) in enumerate(zip(self.param_groups[0]["params"], self._flat_offsets)):
                sd["state"][i] = {"step": torch.tensor(t, dtype=torch.float32),
                                  **{k: b[..., off:off + p.numel()] for k, b in zip(self._state_keys(), self._flat)}}
        return sd


def _check_32bit(optim_bits, percentile_clipping):
    if optim_bits != 32:
        raise NotImplementedError("only 32-bit optimizer state is implemented (SURVEY.md 8f-3)")
    if percentile_clipping != 100:
        raise NotImplementedError("percentile clipping is not supported")


class AdamW(_Optimizer32bit):
    """32-bit AdamW (decoupled weight decay) on CUDA parameters; `is_paged=True` keeps the moments in unified memory.
    State: `state1` = m, `state2` = v."""

    _NAME = "AdamW"
    _STATE_ROWS = (1, 1)

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32, args=None,
                 min_8bit_size=4096, percentile_clipping=100, block_wise=True, is_paged=False, capturable=False):
        _check_32bit(optim_bits, percentile_clipping)
        if amsgrad:
            raise NotImplementedError("amsgrad is not supported")
        if lr < 0 or eps < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1) or weight_decay < 0:
            raise ValueError("invalid AdamW hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), is_paged, capturable)

    def _launch(self, p, g, states, group, step_dev, grad_scale):
        (m, v), (b1, b2) = states, group["betas"]
        check(_lib.load().qb200_adamw32bit_step_dev(ptr(p), DTYPE_CODE[p.dtype], ptr(g), ptr(m), ptr(v), p.numel(), group["lr"], b1, b2,
                                                    group["eps"], group["weight_decay"], ptr(step_dev), ptr(grad_scale),
                                                    stream_ptr(p.device)), "adamw32bit_step_dev")

    def _launch_eager(self, p, g, states, group, step: int):
        (m, v), (b1, b2) = states, group["betas"]
        check(_lib.load().qb200_adamw32bit_step(ptr(p), DTYPE_CODE[p.dtype], ptr(g), ptr(m), ptr(v), p.numel(), group["lr"], b1, b2,
                                                group["eps"], group["weight_decay"], step, 1.0, stream_ptr(p.device)), "adamw32bit_step")


class AdamW32bit(AdamW):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, args=None, min_8bit_size=4096,
                 percentile_clipping=100, block_wise=True, is_paged=False, capturable=False):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, 32, args, min_8bit_size, percentile_clipping, block_wise, is_paged,
                         capturable)


class PagedAdamW(AdamW):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32, args=None,
                 min_8bit_size=4096, percentile_clipping=100, block_wise=True, capturable=False):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, optim_bits, args, min_8bit_size, percentile_clipping, block_wise, True,
                         capturable)


class PagedAdamW32bit(AdamW):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, args=None, min_8bit_size=4096,
                 percentile_clipping=100, block_wise=True, capturable=False):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, 32, args, min_8bit_size, percentile_clipping, block_wise, True,
                         capturable)


class Lion(_Optimizer32bit):
    """32-bit Lion: `p -= lr * sign(b1*m + (1-b1)*g)` after decoupled weight decay, then `m = b2*m + (1-b2)*g`.  One fp32
    state (`state1` = m), so half of AdamW's optimizer memory; `is_paged=True` keeps it in unified memory."""

    _NAME = "Lion"
    _STATE_ROWS = (1,)
    _READS_STEP = False

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, optim_bits=32, args=None, min_8bit_size=4096,
                 percentile_clipping=100, block_wise=True, is_paged=False, capturable=False):
        _check_32bit(optim_bits, percentile_clipping)
        if lr < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1) or weight_decay < 0:
            raise ValueError("invalid Lion hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=betas, weight_decay=weight_decay), is_paged, capturable)

    def _launch(self, p, g, states, group, step_dev, grad_scale):
        (m,), (b1, b2) = states, group["betas"]
        check(_lib.load().qb200_lion32bit_step_dev(ptr(p), DTYPE_CODE[p.dtype], ptr(g), ptr(m), p.numel(), group["lr"], b1, b2,
                                                   group["weight_decay"], ptr(step_dev), ptr(grad_scale), stream_ptr(p.device)),
              "lion32bit_step_dev")


class Lion32bit(Lion):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, args=None, min_8bit_size=4096, percentile_clipping=100,
                 block_wise=True, is_paged=False, capturable=False):
        super().__init__(params, lr, betas, weight_decay, 32, args, min_8bit_size, percentile_clipping, block_wise, is_paged, capturable)


class PagedLion(Lion):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, optim_bits=32, args=None, min_8bit_size=4096,
                 percentile_clipping=100, block_wise=True, capturable=False):
        super().__init__(params, lr, betas, weight_decay, optim_bits, args, min_8bit_size, percentile_clipping, block_wise, True,
                         capturable)


class PagedLion32bit(Lion):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0, args=None, min_8bit_size=4096, percentile_clipping=100,
                 block_wise=True, capturable=False):
        super().__init__(params, lr, betas, weight_decay, 32, args, min_8bit_size, percentile_clipping, block_wise, True, capturable)


class RMSprop(_Optimizer32bit):
    """32-bit RMSprop without momentum or centering: `v = alpha*v + (1-alpha)*g^2`, `p -= lr * g / (sqrt(v) + eps)`, with L2
    weight decay added to the gradient.  State: `state1` = v.  There is no paged form (upstream has none either)."""

    _NAME = "RMSprop"
    _STATE_ROWS = (1,)
    _READS_STEP = False

    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False, optim_bits=32, args=None,
                 min_8bit_size=4096, percentile_clipping=100, block_wise=True, capturable=False):
        _check_32bit(optim_bits, percentile_clipping)
        if momentum != 0:
            raise NotImplementedError("RMSprop with momentum is not supported (the kernel keeps no momentum buffer)")
        if centered:
            raise NotImplementedError("centered RMSprop is not supported (the kernel keeps no gradient average)")
        if alpha == 0:
            raise NotImplementedError("RMSprop with alpha == 0 is not supported")
        if lr < 0 or eps < 0 or not (0 < alpha <= 1) or weight_decay < 0:
            raise ValueError("invalid RMSprop hyper-parameter")
        super().__init__(params, dict(lr=lr, alpha=alpha, eps=eps, weight_decay=weight_decay), False, capturable)

    def _launch(self, p, g, states, group, step_dev, grad_scale):
        (v,) = states
        check(_lib.load().qb200_rmsprop32bit_step_dev(ptr(p), DTYPE_CODE[p.dtype], ptr(g), ptr(v), p.numel(), group["lr"], group["alpha"],
                                                      group["eps"], group["weight_decay"], ptr(step_dev), ptr(grad_scale),
                                                      stream_ptr(p.device)), "rmsprop32bit_step_dev")


class RMSprop32bit(RMSprop):
    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False, args=None, min_8bit_size=4096,
                 percentile_clipping=100, block_wise=True, capturable=False):
        super().__init__(params, lr, alpha, eps, weight_decay, momentum, centered, 32, args, min_8bit_size, percentile_clipping, block_wise,
                         capturable)


class AdEMAMix(_Optimizer32bit):
    """32-bit AdEMAMix (Pagliardini et al., 2024): Adam's bias-corrected fast EMA plus `alpha` times a slow EMA of the
    gradient (`beta3`) over the second moment, with optional linear warm-up of alpha (`t_alpha`) and beta3 (`t_beta3`) and
    decoupled weight decay.  State: `state1` = [2, numel] (fast and slow EMA stacked, as upstream's), `state2` = nu."""

    _NAME = "AdEMAMix"
    _STATE_ROWS = (2, 1)

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha=None, t_beta3=None, eps=1e-8, weight_decay=1e-2,
                 optim_bits=32, min_8bit_size=4096, is_paged=False, capturable=False):
        _check_32bit(optim_bits, 100)
        if (lr < 0 or eps < 0 or alpha < 0 or weight_decay < 0 or len(betas) != 3 or not all(0 <= b < 1 for b in betas)
                or (t_alpha is not None and not t_alpha > 0) or (t_beta3 is not None and not t_beta3 > 0)):
            raise ValueError("invalid AdEMAMix hyper-parameter")
        if t_beta3 is not None and not (betas[0] > 0 and betas[2] > 0):
            raise ValueError("the beta3 schedule (t_beta3) needs beta1 > 0 and beta3 > 0")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), alpha=alpha, t_alpha=t_alpha, t_beta3=t_beta3, eps=eps,
                                      weight_decay=weight_decay), is_paged, capturable)

    def _launch(self, p, g, states, group, step_dev, grad_scale):
        (m, nu), (b1, b2, b3) = states, group["betas"]
        check(_lib.load().qb200_ademamix32bit_step_dev(ptr(p), DTYPE_CODE[p.dtype], ptr(g), ptr(m[0]), ptr(m[1]), ptr(nu), p.numel(),
                                                       group["lr"], b1, b2, b3, group["alpha"], group["t_alpha"] or 0.0,
                                                       group["t_beta3"] or 0.0, group["eps"], group["weight_decay"], ptr(step_dev),
                                                       ptr(grad_scale), stream_ptr(p.device)), "ademamix32bit_step_dev")


class AdEMAMix32bit(AdEMAMix):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha=None, t_beta3=None, eps=1e-8, weight_decay=1e-2,
                 min_8bit_size=4096, is_paged=False, capturable=False):
        super().__init__(params, lr, betas, alpha, t_alpha, t_beta3, eps, weight_decay, 32, min_8bit_size, is_paged, capturable)


class PagedAdEMAMix(AdEMAMix):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha=None, t_beta3=None, eps=1e-8, weight_decay=1e-2,
                 optim_bits=32, min_8bit_size=4096, capturable=False):
        super().__init__(params, lr, betas, alpha, t_alpha, t_beta3, eps, weight_decay, optim_bits, min_8bit_size, True, capturable)


class PagedAdEMAMix32bit(AdEMAMix):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha=None, t_beta3=None, eps=1e-8, weight_decay=1e-2,
                 min_8bit_size=4096, capturable=False):
        super().__init__(params, lr, betas, alpha, t_alpha, t_beta3, eps, weight_decay, 32, min_8bit_size, True, capturable)


class GlobalOptimManager:
    """Name kept for HF's `GlobalOptimManager.get_instance().register_module_override(...)` (8-bit embedding overrides):
    with 32-bit state everywhere there is nothing to override."""

    _instance = None

    @classmethod
    def get_instance(cls):
        if cls._instance is None:
            cls._instance = cls()
        return cls._instance

    def register_module_override(self, module, param_name, config):
        return None

    def register_parameters(self, params):
        return None

    def override_config(self, parameters, key=None, value=None, key_value_dict=None):
        return None
