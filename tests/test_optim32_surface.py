"""CPU tests for the 32-bit Lion, RMSprop and AdEMAMix optimizers: HF Trainer's bitsandbytes factory builds this library's
classes for every 32-bit name and refuses every 8-bit one, upstream's signatures and defaults, every rejected option, and
the C-ABI's argument errors (returned before any launch, so no GPU is needed)."""
import ctypes as ct
import inspect
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Run in a fresh interpreter with the shim first on the path: transformers caches its bitsandbytes probe per process.
# OptimizerContext is built from a plain namespace because TrainingArguments needs accelerate.
_FACTORY_CASE = r"""
import json, types
import torch
import transformers.trainer_optimizer as to

out = {}
for name in to._BITSANDBYTES_OPTIMIZERS:
    name = getattr(name, "value", name)
    args = types.SimpleNamespace(optim=name, adam_beta1=0.9, adam_beta2=0.999, adam_epsilon=1e-8)
    ctx = to.OptimizerContext(args=args, model=None, optimizer_kwargs={"lr": 2e-4}, adam_kwargs={"betas": (0.9, 0.999), "eps": 1e-8},
                              optim_args={})
    cls, kwargs = to._get_bitsandbytes_optimizer(ctx)
    try:
        opt = cls([torch.nn.Parameter(torch.zeros(8))], **kwargs)
        out[name] = {"module": cls.__module__, "cls": cls.__name__, "is_paged": opt.is_paged, "lr": opt.param_groups[0]["lr"]}
    except NotImplementedError as e:
        out[name] = {"module": cls.__module__, "cls": cls.__name__, "error": "NotImplementedError", "msg": str(e)}
print(json.dumps(out))
"""

THIRTY_TWO_BIT = {"paged_adamw_32bit": ("AdamW", True), "lion_32bit": ("Lion", False), "paged_lion_32bit": ("Lion", True),
                  "rmsprop_bnb": ("RMSprop", False), "rmsprop_bnb_32bit": ("RMSprop", False), "ademamix": ("AdEMAMix", False),
                  "paged_ademamix_32bit": ("AdEMAMix", True)}


def test_trainer_factory_builds_every_32bit_optimizer_and_refuses_8bit():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "shims") + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-c", _FACTORY_CASE], capture_output=True, text=True, env=env, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(out) == 15
    for name, res in out.items():
        assert res["module"] == "qlora_b200.optim", (name, res)
        if name in THIRTY_TWO_BIT:
            cls, paged = THIRTY_TWO_BIT[name]
            assert "error" not in res, (name, res)
            assert (res["cls"], res["is_paged"], res["lr"]) == (cls, paged, 2e-4), (name, res)
        else:
            assert "8bit" in name and res["error"] == "NotImplementedError" and "32-bit" in res["msg"], (name, res)
    assert set(THIRTY_TWO_BIT) <= set(out)


def _defaults(cls):
    return {k: v.default for k, v in inspect.signature(cls.__init__).parameters.items() if k not in ("self", "params")}


def test_signatures_and_defaults():
    from qlora_b200 import optim as O

    common = dict(args=None, min_8bit_size=4096, percentile_clipping=100, block_wise=True)
    lion = dict(lr=1e-4, betas=(0.9, 0.99), weight_decay=0, **common)
    assert _defaults(O.Lion) == dict(lion, optim_bits=32, is_paged=False, capturable=False)
    assert _defaults(O.Lion32bit) == dict(lion, is_paged=False, capturable=False)
    assert _defaults(O.PagedLion) == dict(lion, optim_bits=32, capturable=False)
    assert _defaults(O.PagedLion32bit) == dict(lion, capturable=False)
    rms = dict(lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False, **common)
    assert _defaults(O.RMSprop) == dict(rms, optim_bits=32, capturable=False)
    assert _defaults(O.RMSprop32bit) == dict(rms, capturable=False)
    ade = dict(lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, t_alpha=None, t_beta3=None, eps=1e-8, weight_decay=1e-2, min_8bit_size=4096)
    assert _defaults(O.AdEMAMix) == dict(ade, optim_bits=32, is_paged=False, capturable=False)
    assert _defaults(O.AdEMAMix32bit) == dict(ade, is_paged=False, capturable=False)
    assert _defaults(O.PagedAdEMAMix) == dict(ade, optim_bits=32, capturable=False)
    assert _defaults(O.PagedAdEMAMix32bit) == dict(ade, capturable=False)
    # positional order is upstream's
    assert list(_defaults(O.Lion))[:4] == ["lr", "betas", "weight_decay", "optim_bits"]
    assert list(_defaults(O.RMSprop))[:7] == ["lr", "alpha", "eps", "weight_decay", "momentum", "centered", "optim_bits"]
    assert list(_defaults(O.AdEMAMix))[:9] == ["lr", "betas", "alpha", "t_alpha", "t_beta3", "eps", "weight_decay", "optim_bits",
                                               "min_8bit_size"]

    p = torch.nn.Parameter(torch.zeros(8))
    for cls, paged in ((O.Lion, False), (O.Lion32bit, False), (O.PagedLion, True), (O.PagedLion32bit, True), (O.RMSprop, False),
                       (O.RMSprop32bit, False), (O.AdEMAMix, False), (O.AdEMAMix32bit, False), (O.PagedAdEMAMix, True),
                       (O.PagedAdEMAMix32bit, True)):
        opt = cls([p])
        assert opt.is_paged is paged and not opt.capturable and isinstance(opt, torch.optim.Optimizer), cls
    g = O.AdEMAMix([p], t_alpha=100, t_beta3=200).param_groups[0]
    assert (g["betas"], g["alpha"], g["t_alpha"], g["t_beta3"], g["weight_decay"]) == ((0.9, 0.999, 0.9999), 5.0, 100, 200, 1e-2)
    assert issubclass(O.PagedLion32bit, O.Lion) and issubclass(O.RMSprop32bit, O.RMSprop) and issubclass(O.PagedAdEMAMix32bit, O.AdEMAMix)
    # the shim exposes the same classes under bitsandbytes.optim
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    from bitsandbytes.optim import AdEMAMix, Lion, PagedAdEMAMix32bit, PagedLion32bit, RMSprop  # noqa: F401
    assert Lion is O.Lion and RMSprop is O.RMSprop and AdEMAMix is O.AdEMAMix


def test_rejected_options():
    from qlora_b200 import optim as O

    p = torch.nn.Parameter(torch.zeros(8))
    not_impl = [lambda: O.Lion([p], optim_bits=8), lambda: O.PagedLion([p], optim_bits=8), lambda: O.Lion([p], percentile_clipping=5),
                lambda: O.RMSprop([p], optim_bits=8), lambda: O.RMSprop([p], percentile_clipping=5), lambda: O.RMSprop([p], momentum=0.9),
                lambda: O.RMSprop([p], centered=True), lambda: O.RMSprop([p], alpha=0), lambda: O.AdEMAMix([p], optim_bits=8),
                lambda: O.PagedAdEMAMix([p], optim_bits=8)]
    for i, make in enumerate(not_impl):
        with pytest.raises(NotImplementedError):
            make()
            pytest.fail(f"case {i}")
    bad = [lambda: O.Lion([p], lr=-1), lambda: O.Lion([p], betas=(1.0, 0.99)), lambda: O.Lion([p], betas=(0.9, -0.1)),
           lambda: O.Lion([p], weight_decay=-1), lambda: O.RMSprop([p], lr=-1), lambda: O.RMSprop([p], eps=-1),
           lambda: O.RMSprop([p], alpha=1.5), lambda: O.RMSprop([p], alpha=-0.5), lambda: O.RMSprop([p], weight_decay=-1),
           lambda: O.AdEMAMix([p], lr=-1), lambda: O.AdEMAMix([p], eps=-1), lambda: O.AdEMAMix([p], alpha=-1),
           lambda: O.AdEMAMix([p], weight_decay=-1), lambda: O.AdEMAMix([p], betas=(0.9, 0.999)),
           lambda: O.AdEMAMix([p], betas=(0.9, 0.999, 1.0)), lambda: O.AdEMAMix([p], t_alpha=0),
           lambda: O.AdEMAMix([p], t_beta3=-5), lambda: O.AdEMAMix([p], betas=(0.0, 0.999, 0.9999), t_beta3=10)]
    for i, make in enumerate(bad):
        with pytest.raises(ValueError):
            make()
            pytest.fail(f"case {i}")
    for cls in (O.Lion, O.PagedLion32bit, O.RMSprop, O.AdEMAMix, O.PagedAdEMAMix32bit):
        opt = cls([p])
        p.grad = torch.ones(8)
        with pytest.raises(RuntimeError, match="CUDA"):
            opt.step()   # CPU parameter: no CPU fallback
        with pytest.raises(ValueError, match="capturable"):
            opt.step_flat(p.detach(), p.grad)


def test_argument_errors_return_einval_before_any_launch():
    """Run on a thread of its own: the error message is thread-local, so the messages set here stay out of other tests."""
    import threading

    failure = []

    def run():
        try:
            _argument_errors()
        except BaseException as e:   # noqa: BLE001 (re-raised on the test's thread)
            failure.append(e)

    t = threading.Thread(target=run)
    t.start()
    t.join()
    if failure:
        raise failure[0]


def _argument_errors():
    from qlora_b200 import _lib

    lib = _lib.load()
    buf = (ct.c_char * 256)()
    q = ct.cast(buf, ct.c_void_p)

    def err():
        return lib.qb200_last_error()

    lion = lambda p, dt, g, m, n: lib.qb200_lion32bit_step_dev(p, dt, g, m, n, 1e-4, 0.9, 0.99, 0.0, None, None, None)  # noqa: E731
    rms = lambda p, dt, g, v, n: lib.qb200_rmsprop32bit_step_dev(p, dt, g, v, n, 1e-2, 0.99, 1e-8, 0.0, None, None, None)  # noqa: E731

    def ade(p, dt, g, m1, m2, nu, n, step=q, t_alpha=0.0, t_beta3=0.0):
        return lib.qb200_ademamix32bit_step_dev(p, dt, g, m1, m2, nu, n, 1e-3, 0.9, 0.999, 0.9999, 5.0, t_alpha, t_beta3, 1e-8, 0.01, step,
                                                None, None)

    for fn, nargs, what in ((lion, 3, b"lion32bit"), (rms, 3, b"rmsprop32bit")):
        args = [q] * nargs
        for i in range(nargs):   # each of p, g and the state missing
            a = list(args)
            a[i] = None
            assert fn(a[0], 2, a[1], a[2], 64) == -1 and what in err() and b"null pointer" in err()
        assert fn(q, 2, q, q, -1) == -1 and b"n < 0" in err()
        assert fn(q, 3, q, q, 64) == -1 and b"dtype" in err()
        assert fn(q, -1, q, q, 64) == -1 and b"dtype" in err()
    for i in range(5):   # p, g, m1, m2, nu
        a = [q] * 5
        a[i] = None
        assert ade(a[0], 2, a[1], a[2], a[3], a[4], 64) == -1 and b"ademamix32bit" in err() and b"null pointer" in err()
    assert ade(q, 2, q, q, q, q, 64, step=None) == -1 and b"null pointer" in err()   # AdEMAMix reads the step count
    assert ade(q, 2, q, q, q, q, -1) == -1 and b"n < 0" in err()
    assert ade(q, 7, q, q, q, q, 64) == -1 and b"dtype" in err()
    assert ade(q, 2, q, q, q, q, 64, t_alpha=-1.0) == -1 and b"t_alpha" in err()
    assert ade(q, 2, q, q, q, q, 64, t_beta3=-3.0) == -1 and b"t_beta3" in err()
    assert ade(q, 2, q, q, q, q, 64, t_alpha=float("nan")) == -1 and b"t_alpha" in err()
    # n == 0 is a valid empty update: nothing is launched, so no GPU is needed either
    assert lion(q, 2, q, q, 0) == 0 and rms(q, 0, q, q, 0) == 0 and ade(q, 1, q, q, q, q, 0) == 0
