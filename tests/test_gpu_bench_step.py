"""The training step `bench.py` times, checked against a float64 restatement of the same step (tests/step_reference.py).

The tiny Llama-QLoRA model is built and stepped the way `bench.py` runs the 7B one: grouped fused launches, adapter
gradients accumulated in place into `FlatGradSync`'s flat bf16 buffer, parameters in one flat buffer updated by
`PagedAdamW32bit.step_flat` with the device-side clip coefficient, checkpointing, one dropout seed bump per micro-step,
`loss / accum`, deterministic algorithms.  LoRA r = 64, alpha = 16 (scaling 0.25, so a dropped or doubled scaling shows).

The reference sees the same bf16 constants (the C oracle's dequantized weights, the embeddings, lm_head, RoPE tables and
adapters), so every difference is a rounding of the GPU step.  Its error is set against the same step run unfused
(dequantize + cuBLAS, peft-form LoRA, torch elementwise ops, gradients through autograd), measured on the same reference.

Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W): relative Frobenius error of the accumulated adapter gradients
of the first optimizer step against float64, largest over the 14 dA (dB) tensors of each case, library arm / unfused arm:

    case                     dA               dB
    fused_p0_accum1          1.03e-2 / 1.19e-2   1.02e-2 / 1.20e-2
    fused_p0.1_accum2        1.09e-2 / 1.21e-2   1.08e-2 / 1.24e-2
    scratch_p0_accum2        1.05e-2 / 1.20e-2   1.03e-2 / 1.19e-2
    scratch_p0.1_accum2      1.09e-2 / 1.19e-2   1.07e-2 / 1.22e-2
    scratch_zero_b           (exactly 0)         1.02e-2 / 1.05e-2
    scratch_norm_out_fp32    1.05e-2 / 1.18e-2   1.07e-2 / 1.17e-2

The second step's errors are the same (0.99e-2 to 1.11e-2).  The micro-step losses are within 2.2e-5 (library) and 1.8e-5
(unfused) relative.  The ceilings below are about twice the unfused arm's largest error.  The negative controls show that
they still reject a doubled scaling (error 0.50 to 0.67), a lost micro-step (1.03 to 1.12), the masks of the neighbouring
call site (0.49 to 0.51) and q's dA written into k's rows (1.44 to 1.46), by 20x or more.
"""
import math

import numpy as np
import pytest
import torch

import step_reference as R
from gpu_helpers import oracle_weight

pytestmark = pytest.mark.gpu

CEIL_DA = 2.5e-2    # relative Frobenius error of each dA
CEIL_DB = 2.5e-2    # ... and of each dB
CEIL_LOSS = 5e-5    # relative error of each micro-step's loss

CASES = {
    "fused_p0_accum1": dict(seq=1000, p=0.0, accum=1),
    "fused_p0.1_accum2": dict(seq=1000, p=0.1, accum=2),
    "scratch_p0_accum2": dict(seq=2048, p=0.0, accum=2),
    "scratch_p0.1_accum2": dict(seq=2048, p=0.1, accum=2),
    "scratch_zero_b": dict(seq=2048, p=0.0, accum=1, zero_b=True),
    "scratch_norm_out_fp32": dict(seq=2048, p=0.1, accum=1, norm_out_fp32=True),
}
LR, BETAS, EPS = 2e-4, (0.9, 0.999), 1e-8


@pytest.fixture(scope="module")
def H():
    assert torch.cuda.is_available()
    import harness.llama_qlora as H
    from harness import fused_ops

    fused_ops.build()
    assert fused_ops.available()
    return H


@pytest.fixture
def deterministic(monkeypatch):
    """The attention backward and cuBLAS in their deterministic forms, as bench.py runs them."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev, prev_fill = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    torch.backends.cuda.matmul.allow_tf32 = True
    yield
    torch.use_deterministic_algorithms(prev)
    torch.utils.deterministic.fill_uninitialized_memory = prev_fill
    torch.backends.cuda.matmul.allow_tf32 = prev_tf32


def _bench_settings(mp, H, fused: bool):
    """bench.py's module globals (fused = the default arm; unfused = `--impl unfused`, with gradients through autograd)."""
    from qlora_b200 import autograd as qauto
    from qlora_b200 import lora

    mp.setattr(lora, "ACCUMULATE_ADAPTER_GRADS_IN_PLACE", fused)
    mp.setattr(H, "GROUP_LINEARS", fused)
    mp.setattr(H, "USE_FUSED_OPS", fused)
    mp.setattr(qauto, "USE_FUSED", fused)
    if not fused:   # torch's elementwise ops everywhere, but the same seeded masks (torch's nn.Dropout would draw others)
        mp.setattr(H.LoRALinear4bit, "lora_input", _seeded_lora_input)


def _seeded_lora_input(self, x):
    from harness import fused_ops

    if self.p <= 0.0 or not self.training:
        return None
    return fused_ops.seeded_dropout(x.to(torch.bfloat16), self.p, self._seed[0], self.salt)


def _lora_modules(H, model):
    return [(li, n, getattr(layer, n)) for li, layer in enumerate(model.layers) for n in R.LINEARS]


class BenchStep:
    """The tiny model, its optimizer and flat buffers, and bench.py's micro-step body with the flat gradient copied ahead
    of the optimizer."""

    def __init__(self, H, cfg, fused=True, salts=None):
        from harness.dp import FlatGradSync
        import qlora_b200 as q

        self.H, self.cfg = H, cfg
        shape = H.SHAPES["tiny"]
        dev = torch.device("cuda")
        model = H.LlamaQLoRA(shape, dev, lora_r=64, lora_alpha=16, lora_dropout=cfg["p"], seed=1234, double_quant=True,
                             grad_checkpointing=True, norm_out_fp32=cfg.get("norm_out_fp32", False)).train()
        gen = torch.Generator(device="cuda").manual_seed(99)
        for li, n, m in _lora_modules(H, model):
            if not cfg.get("zero_b"):
                torch.nn.init.normal_(m.lora_B.weight, std=0.05, generator=gen)
            if not fused:
                m.fused = False
            if salts is not None:
                m.salt = salts[(li, n)]
        self.model = model
        self.names = [n for n, _ in model._trainable_named()]
        params = model.trainable_parameters()
        self.opt = q.optim.PagedAdamW32bit(params, lr=LR, betas=BETAS, weight_decay=0.0, capturable=True)
        self.gsync = FlatGradSync(params, 1, layer_of=model.trainable_parameter_layers(), n_buckets=1, overlap=True, flat_params=True)
        self.sizes = [p.numel() for p in params]
        self.shapes = [tuple(p.shape) for p in params]
        self.accum = cfg["accum"]
        self.batches = [H.synthetic_batch(shape, cfg["seq"], seed=50 + j) for j in range(2 * self.accum)]
        self.ids = self.batches[0][0].to(dev)
        self.labels = self.batches[0][1].to(dev)
        self.loss = torch.zeros((), device=dev)
        self.clip = torch.ones((), device=dev)
        self.grad_seen = torch.zeros_like(self.gsync.flat)   # the gradient step_flat was given

    def body(self, first, last):
        model, gsync = self.model, self.gsync
        if first:
            gsync.zero()
        model.dropout_seed.add_(1)
        loss = model(self.ids, self.labels)
        if self.accum > 1:
            loss = loss / self.accum
        loss.backward()
        self.loss.copy_(loss.detach())
        if last:
            gsync.finish()
            self.grad_seen.copy_(gsync.flat)
            torch.clamp(0.3 / (torch.linalg.vector_norm(gsync.flat, dtype=torch.float32) + 1e-6), max=1.0, out=self.clip)
            self.opt.step_flat(gsync.flat_param, gsync.flat, grad_scale=self.clip)

    def kinds(self):
        return [(mi == 0, mi == self.accum - 1) for mi in range(self.accum)]

    def step(self, k, graphs=None):
        """Optimizer step k (batches k*accum ...): per micro-step (loss, dropout seed); then the gradient, clip coefficient
        and parameters after the step."""
        micro = []
        for mi, kd in enumerate(self.kinds()):
            ids, labels = self.batches[k * self.accum + mi]
            self.ids.copy_(ids)
            self.labels.copy_(labels)
            if graphs:
                graphs[kd].replay()
            else:
                self.body(*kd)
            micro.append((self.loss.clone(), int(self.model.dropout_seed.item())))
        torch.cuda.synchronize()
        return dict(micro=micro, grad=self.grad_seen.clone(), flat_grad=self.gsync.flat.clone(), clip=self.clip.clone(),
                    params=self.gsync.flat_param.clone())

    def split(self, flat):
        return dict(zip(self.names, (t.view(s) for t, s in zip(flat.split(self.sizes), self.shapes))))

    def reference_model(self, c_oracle, scaling_mult=1.0, salt_shift=0):
        H, model = self.H, self.model
        shape = H.SHAPES["tiny"]
        weights, salts = {}, {}
        for li, n, m in _lora_modules(H, model):
            w = m.base_layer.weight
            weights[(li, n)] = torch.from_numpy(oracle_weight(w.data, w.quant_state, c_oracle)).double()
            salts[(li, n)] = m.salt + salt_shift
        cos, sin = H._rope_tables(self.cfg["seq"], shape.hidden // shape.heads, shape.rope_theta, "cuda")
        f64 = lambda t: t.detach().double().cpu()   # noqa: E731
        return R.RefModel(weights=weights, norms={(li, k): f64(getattr(layer, k + ("_layernorm" if k == "input" else "_attention_layernorm")).weight)
                                                  for li, layer in enumerate(model.layers) for k in ("input", "post")},
                          final_norm=f64(model.norm.weight), embed=f64(model.embed_tokens.weight), lm_head=f64(model.lm_head.weight),
                          cos=f64(cos[:, 0]), sin=f64(sin[:, 0]), heads=shape.heads, eps=shape.rms_eps,
                          scaling=model.layers[0].q_proj.scaling * scaling_mult, p=self.cfg["p"], salts=salts)

    def salts(self):
        return {(li, n): m.salt for li, n, m in _lora_modules(self.H, self.model)}


def reference_step(bs: BenchStep, ref: R.RefModel, adapters: dict, k: int, seeds):
    """Float64 micro-step losses (divided by accum) and per-micro-step gradients (divided by accum) of optimizer step k."""
    losses, grads = [], []
    for mi in range(bs.accum):
        ids, labels = bs.batches[k * bs.accum + mi]
        loss, g = R.micro_step(ref, adapters, ids, labels, seeds[mi])
        losses.append(loss / bs.accum)
        grads.append({n: t / bs.accum for n, t in g.items()})
    return losses, grads


def _sum(grads):
    return {n: sum(g[n] for g in grads) for n in grads[0]}


def rel_errors(got: dict, ref: dict) -> dict:
    """{name: ||got - ref||_F / ||ref||_F}, None where the reference is exactly zero."""
    out = {}
    for n, r in ref.items():
        rn = float(r.norm())
        out[n] = None if rn == 0.0 else float((got[n].double().cpu() - r).norm()) / rn
    return out


def ceiling(name):
    return CEIL_DA if "lora_A" in name else CEIL_DB


def _f64(flat_dict):
    return {n: t.detach().double().cpu() for n, t in flat_dict.items()}


_RUNS = {}


def run_case(H, c_oracle, monkeypatch, case):
    """Both arms of one case, two optimizer steps each, and the float64 references of both steps (cached per module)."""
    if case in _RUNS:
        return _RUNS[case]
    cfg = CASES[case]
    out = {}
    with monkeypatch.context() as mp:
        _bench_settings(mp, H, fused=True)
        ours = BenchStep(H, cfg)
        p0 = ours.gsync.flat_param.clone()
        a0 = _f64(ours.split(p0))
        out["ours"] = [ours.step(0), ours.step(1)]
    with monkeypatch.context() as mp:
        _bench_settings(mp, H, fused=False)
        unf = BenchStep(H, cfg, fused=False, salts=ours.salts())
        assert torch.equal(unf.gsync.flat_param, p0) and unf.names == ours.names
        out["unfused"] = [unf.step(0)]
    ref = ours.reference_model(c_oracle)
    seeds0 = [s for _, s in out["ours"][0]["micro"]]
    seeds1 = [s for _, s in out["ours"][1]["micro"]]
    a1 = _f64(ours.split(out["ours"][0]["params"]))
    out.update(bs=ours, ref=ref, p0=p0, a0=a0, a1=a1, seeds=(seeds0, seeds1),
               step0=reference_step(ours, ref, a0, 0, seeds0), step1=reference_step(ours, ref, a1, 1, seeds1))
    _RUNS[case] = out
    return out


def _worst(errs: dict) -> float:
    """Largest error over the tensors, in units of each tensor's ceiling."""
    return max(e / ceiling(n) for n, e in errs.items() if e is not None)


@pytest.mark.parametrize("case", sorted(CASES))
def test_loss_and_gradients_match_float64(H, c_oracle, deterministic, monkeypatch, case):
    from qlora_b200 import _lib

    cfg = CASES[case]
    assert (_lib.load().qb200_nf4_linear_scratch_size(1, cfg["seq"], 256, 256, 0) > 0) == (cfg["seq"] == 2048)
    r = run_case(H, c_oracle, monkeypatch, case)
    bs, accum = r["bs"], cfg["accum"]
    assert r["seeds"] == (list(range(1, accum + 1)), list(range(accum + 1, 2 * accum + 1)))   # one bump per micro-step
    ref_losses, ref_grads = r["step0"]
    for (loss, _), want in zip(r["ours"][0]["micro"], ref_losses):
        assert abs(float(loss) - want) <= CEIL_LOSS * abs(want), (float(loss), want)
    got = bs.split(r["ours"][0]["grad"])
    errs = rel_errors(got, _sum(ref_grads))
    assert len(errs) == 28
    for n, e in errs.items():
        if cfg.get("zero_b") and "lora_A" in n:   # B = 0: G = s dY.B = 0, so dA is exactly zero
            assert e is None and not got[n].any(), n
        else:
            assert e is not None and e <= ceiling(n), (n, e)


@pytest.mark.parametrize("case", sorted(CASES))
def test_error_is_within_the_unfused_arms(H, c_oracle, deterministic, monkeypatch, case):
    """The library's step is no further from float64 than the unfused step (dequantize + cuBLAS + peft-form LoRA)."""
    r = run_case(H, c_oracle, monkeypatch, case)
    bs = r["bs"]
    want = _sum(r["step0"][1])
    ours = rel_errors(bs.split(r["ours"][0]["grad"]), want)
    unfused = rel_errors(bs.split(r["unfused"][0]["grad"]), want)
    for n, e in ours.items():
        if e is not None:
            assert e <= 1.5 * unfused[n] + 1e-3, (n, e, unfused[n])
            assert unfused[n] <= ceiling(n), (n, unfused[n])


def _bf16(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(x).to(torch.bfloat16).double().numpy()


def adamw_f64(p_old, grads, clips):
    """The update of the last of len(grads) AdamW steps from zero moments, in float64 with the fp32 hyper-parameters the
    kernel reads (weight decay 0)."""
    f32 = lambda v: float(np.float32(v))   # noqa: E731
    lr, b1, b2, eps = f32(LR), f32(BETAS[0]), f32(BETAS[1]), f32(EPS)
    m = v = 0.0
    for g, c in zip(grads, clips):
        gi = c * g
        m = b1 * m + (1 - b1) * gi
        v = b2 * v + (1 - b2) * gi * gi
    t = len(grads)
    c1, c2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
    return (-lr * c2 / c1) * m / (np.sqrt(v) + eps * c2)


def update_matches(p_new, p_old, upd, t):
    """Element-wise: p_new is a bf16 rounding of a value within the kernel's fp32 error `tol` of p_old + upd: the bf16
    rounding of p_old + upd itself, unless that lies within `tol` of a rounding boundary.  `tol` is 2^-20 of the terms'
    magnitude plus, on the update, the error of the fp32 bias corrections 1 - beta^t: a few fp32 ulps of beta^t (powf)
    over 1 - beta^t, which cancels (beta2 = 0.999: about 1e-4 of the update at t = 2, none at t = 1).  Where p_old and the
    update nearly cancel, `tol` can span a few ulps of the small result."""
    b1, b2 = float(np.float32(BETAS[0])), float(np.float32(BETAS[1]))
    corr = 0.0 if t == 1 else 2.0 ** -22 * (b1 ** t / (1 - b1 ** t) + b2 ** t / (1 - b2 ** t))
    want = p_old + upd
    tol = 2.0 ** -20 * (np.abs(p_old) + np.abs(upd)) + corr * np.abs(upd)
    return (p_new >= _bf16(want - tol)) & (p_new <= _bf16(want + tol))   # bf16 rounding is monotone


@pytest.mark.parametrize("case", sorted(CASES))
def test_optimizer_update_matches_float64(H, c_oracle, deterministic, monkeypatch, case):
    """step_flat, the device-side clip coefficient and the flat parameter views together: every adapter weight after each
    of two steps is the bf16 rounding of the float64 AdamW update computed from the GPU's own gradient and clip."""
    r = run_case(H, c_oracle, monkeypatch, case)
    steps = r["ours"]
    gs = [s["grad"].double().cpu().numpy() for s in steps]
    clips = [float(s["clip"]) for s in steps]
    for g, c in zip(gs, clips):
        want = min(1.0, 0.3 / (np.linalg.norm(g) + 1e-6))
        assert abs(c - want) <= 1e-5 * want, (c, want)
    p_prev = r["p0"].double().cpu().numpy()
    for k, s in enumerate(steps):
        p_new = s["params"].double().cpu().numpy()
        upd = adamw_f64(p_prev, gs[:k + 1], clips[:k + 1])
        ok = update_matches(p_new, p_prev, upd, k + 1)
        bad = np.flatnonzero(~ok)[:4]
        assert ok.all(), (k, int((~ok).sum()), bad, p_prev[bad], upd[bad], p_new[bad])
        moved = gs[k] != 0
        assert (p_new[moved] != p_prev[moved]).mean() > 0.5, k   # an update of ~lr is about one bf16 ulp of a 0.05 weight
        assert not update_matches(p_prev, p_prev, upd, k + 1).all()   # a step that changed nothing fails the check
        p_prev = p_new


@pytest.mark.parametrize("case", sorted(CASES))
def test_second_step_gradients_match_float64(H, c_oracle, deterministic, monkeypatch, case):
    """The second optimizer step, against float64 from the parameters the first one produced: a gradient buffer that is not
    zeroed between steps, or an in-place sink that still points at old storage, fails here."""
    r = run_case(H, c_oracle, monkeypatch, case)
    bs = r["bs"]
    ref_losses, ref_grads = r["step1"]
    for (loss, _), want in zip(r["ours"][1]["micro"], ref_losses):
        assert abs(float(loss) - want) <= CEIL_LOSS * abs(want), (float(loss), want)
    for n, e in rel_errors(bs.split(r["ours"][1]["grad"]), _sum(ref_grads)).items():
        assert e is not None and e <= ceiling(n), (n, e)


@pytest.mark.parametrize("case", sorted(CASES))
def test_negative_controls_exceed_the_bounds(H, c_oracle, deterministic, monkeypatch, case):
    """Float64 references of wrong steps are rejected by the ceilings with a margin of 3: scaling doubled, one micro-step
    left out, masks of the neighbouring call site, q's and k's dA swapped."""
    r = run_case(H, c_oracle, monkeypatch, case)
    bs, cfg = r["bs"], CASES[case]
    got = bs.split(r["ours"][0]["grad"])
    seeds0 = r["seeds"][0]
    right = _sum(r["step0"][1])
    _, doubled = reference_step(bs, bs.reference_model(c_oracle, scaling_mult=2.0), r["a0"], 0, seeds0)
    assert _worst(rel_errors(got, _sum(doubled))) >= 3
    if cfg["accum"] > 1:
        assert _worst(rel_errors(got, _sum(r["step0"][1][:-1]))) >= 3
    if cfg["p"] > 0:
        _, shifted = reference_step(bs, bs.reference_model(c_oracle, salt_shift=1), r["a0"], 0, seeds0)
        assert _worst(rel_errors(got, _sum(shifted))) >= 3
    if not cfg.get("zero_b"):
        swapped = dict(right)
        for li in range(len(bs.model.layers)):
            q, k = R.adapter_name(li, "q_proj", "A"), R.adapter_name(li, "k_proj", "A")
            swapped[q], swapped[k] = right[k], right[q]
        assert _worst(rel_errors(got, swapped)) >= 3


@pytest.mark.parametrize("case", ["fused_p0.1_accum2", "scratch_p0.1_accum2"])
def test_cuda_graph_replay_equals_eager(H, deterministic, monkeypatch, case):
    """One graph per micro-step kind, as bench.py captures them, replayed for two optimizer steps from a restored
    pre-warm-up state: loss, gradients, clip coefficient and parameters equal an eager run from the same state bit for bit."""
    with monkeypatch.context() as mp:
        _bench_settings(mp, H, fused=True)
        bs = BenchStep(H, CASES[case])
        snap = (bs.gsync.flat_param.clone(), bs.gsync.flat.clone(), bs.model.dropout_seed.clone())
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                for kd in bs.kinds():
                    bs.body(*kd)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graphs = {}
        for kd in bs.kinds():
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                bs.body(*kd)
            graphs[kd] = g

        def restore():   # in place: the graphs hold these addresses
            bs.gsync.flat_param.copy_(snap[0])
            bs.gsync.flat.copy_(snap[1])
            bs.model.dropout_seed.copy_(snap[2])
            for t in bs.opt._flat:
                t.zero_()
            bs.opt._step_dev.zero_()
            torch.cuda.synchronize()

        restore()
        eager = [bs.step(0), bs.step(1)]
        restore()
        replayed = [bs.step(0, graphs), bs.step(1, graphs)]
    assert not torch.equal(eager[1]["params"], snap[0])
    for e, g in zip(eager, replayed):
        assert [(float(l), s) for l, s in e["micro"]] == [(float(l), s) for l, s in g["micro"]]
        for key in ("grad", "flat_grad", "clip", "params"):
            assert torch.equal(e[key], g[key]), key
