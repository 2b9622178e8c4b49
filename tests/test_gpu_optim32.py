"""GPU tests of the 32-bit Lion, RMSprop and AdEMAMix optimizers (qlora_b200/csrc/optim32.cu) against the fp32 restatements
in tests/optim_oracle.py, a float64 restatement, torch's RMSprop, and each other across paging, resume, CUDA-graph replay
and the flat one-launch form; and the benchmarked training step with Lion and AdEMAMix in place of AdamW."""
import math

import numpy as np
import pytest
import torch

import optim_oracle as oo
from test_gpu_bench_step import CASES, LR, BenchStep, H, _bench_settings, deterministic  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu

HP = {"lion": dict(lr=1e-3, betas=(0.9, 0.99), weight_decay=0.01),
      "rmsprop": dict(lr=1e-3, alpha=0.99, eps=1e-8, weight_decay=0.01),
      "ademamix": dict(lr=1e-3, betas=(0.9, 0.999, 0.9999), alpha=5.0, eps=1e-8, weight_decay=0.01)}
# RMSprop has no paged form (upstream has none either)
RULE_PAGED = [("lion", False), ("lion", True), ("rmsprop", False), ("ademamix", False), ("ademamix", True)]
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def make(rule, params, paged=False, capturable=False, **kw):
    import qlora_b200 as q

    hp = dict(HP[rule], **kw)
    if rule == "lion":
        return q.optim.Lion(params, is_paged=paged, capturable=capturable, **hp)
    if rule == "rmsprop":
        assert not paged
        return q.optim.RMSprop(params, capturable=capturable, **hp)
    return q.optim.AdEMAMix(params, is_paged=paged, capturable=capturable, **hp)


def gpu_state(rule, st):
    """The fp32 state of one parameter as numpy arrays, in the oracle's argument order."""
    if rule == "ademamix":
        return [st["state1"][0].cpu().numpy(), st["state1"][1].cpu().numpy(), st["state2"].cpu().numpy()]
    return [st["state1"].cpu().numpy()]


def oracle_step(rule, p, g, state, step, hp, gnorm_scale=1.0):
    if rule == "lion":
        p2, m = oo.lion32bit_step(p, g, state[0], hp["lr"], *hp["betas"], hp["weight_decay"], gnorm_scale)
        return p2, [m]
    if rule == "rmsprop":
        p2, v = oo.rmsprop32bit_step(p, g, state[0], hp["lr"], hp["alpha"], hp["eps"], hp["weight_decay"], gnorm_scale)
        return p2, [v]
    p2, m1, m2, nu = oo.ademamix32bit_step(p, g, *state, hp["lr"], *hp["betas"], hp["alpha"], hp["eps"], hp["weight_decay"], step,
                                           hp.get("t_alpha"), hp.get("t_beta3"), gnorm_scale)
    return p2, [m1, m2, nu]


def _round(x, dtype):
    return torch.from_numpy(np.asarray(x, np.float32)).to(dtype).float().numpy()


def _check_against_oracle(rule, dtype, paged, n, steps=3, **kw):
    torch.manual_seed(0)
    hp = dict(HP[rule], **kw)
    p0 = (torch.randn(n) * 0.1).to(dtype)
    p = torch.nn.Parameter(p0.clone().cuda())
    opt = make(rule, [p], paged, **kw)
    pr = p0.float().numpy().copy()
    state = [np.zeros(n, np.float32) for _ in range(3 if rule == "ademamix" else 1)]
    for step in range(1, steps + 1):
        g = (torch.randn(n) * 0.01).to(dtype)
        g[:7] = 0   # zero gradients: Lion's sign(0) on the first step
        p.grad = g.cuda()
        opt.step()
        pr, state = oracle_step(rule, pr, g.float().numpy(), state, step, hp)
        pr = _round(pr, dtype)   # the parameter is stored in `dtype` between steps
        got_state = gpu_state(rule, opt.state[p])
        got = p.detach().float().cpu().numpy()
        if rule in ("lion", "rmsprop"):   # correctly rounded fp32 operations only: bitwise
            for a, b in zip(got_state, state):
                assert np.array_equal(a, b), step
            assert np.array_equal(got, pr), (step, int((got != pr).sum()))
        else:                             # the AdamW test's tolerances
            for a, b in zip(got_state, state):
                assert np.allclose(a, b, rtol=1e-6, atol=1e-12), step
            if dtype == torch.float32:
                assert np.allclose(got, pr, rtol=2e-6, atol=1e-9), step
            else:   # identical up to one rounding step of the storage dtype
                ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
                assert np.all(np.abs(got - pr) <= ulp * np.maximum(np.abs(pr), 1e-3) * 1.01), step
            state = got_state   # carry the GPU's state on (its small differences are not the next step's subject)
    assert float(opt.state[p]["step"]) == steps
    if paged:
        assert id(p) in opt._paged and opt.state[p]["state1"].data_ptr() == opt._paged[id(p)][0].ptr


@pytest.mark.parametrize("n", [64 * 1000 + 37, 64 * 1000 + 36])   # odd (element-wise AdEMAMix) / multiple of 4, vector tail
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rule,paged", RULE_PAGED)
def test_matches_oracle(rule, paged, dtype, n):
    _check_against_oracle(rule, dtype, paged, n)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("paged", [False, True])
def test_ademamix_schedules_match_oracle(dtype, paged):
    """t_alpha = t_beta3 = 2: step 1 is before the end of both warm-ups, step 2 at it, steps 3 and 4 after it."""
    _check_against_oracle("ademamix", dtype, paged, 64 * 100 + 4, steps=4, t_alpha=2, t_beta3=2)
    c = [oo.ademamix_step_scalars(t, 0.9, 0.999, 0.9999, 5.0, 2, 2) for t in (1, 2, 3)]
    assert c[0][2] == np.float32(2.5) and c[1][2] == c[2][2] == np.float32(5.0)
    assert c[0][3] < c[1][3] == c[2][3] == np.float32(0.9999)


def _f64_update(rule, p, g, state, step, hp):
    """The exact update of one step from the GPU's own previous state, in float64 with the fp32 hyper-parameters, and an
    element-wise bound on a correctly implemented fp32 kernel's distance from it."""
    f = lambda v: float(np.float32(v))   # noqa: E731
    lr, wd = f(hp["lr"]), f(hp["weight_decay"])
    u = 2.0 ** -24
    if rule == "lion":
        b1, b2 = f(hp["betas"][0]), f(hp["betas"][1])
        c = b1 * state[0] + (1 - b1) * g
        pd = p * (1 - lr * wd) if wd > 0 else p
        p64 = pd - lr * np.sign(c)
        m64 = b2 * state[0] + (1 - b2) * g
        tol = 4 * u * (np.abs(p) + lr)
        sure = np.abs(c) > 8 * u * (np.abs(b1 * state[0]) + np.abs((1 - b1) * g))   # sign decided beyond fp32 rounding
        return p64, [m64], tol, [4 * u * (np.abs(b2 * state[0]) + np.abs((1 - b2) * g))], sure
    if rule == "rmsprop":
        al, eps = f(hp["alpha"]), f(hp["eps"])
        gw = g + wd * p
        v64 = al * state[0] + (1 - al) * gw * gw
        upd = lr * gw / (np.sqrt(v64) + eps)
        # g + wd*p can cancel: the fp32 rounding of wd*p then dominates gw's error, which reaches p through lr / (sqrt(v) + eps)
        gw_err = 2 * u * (np.abs(wd * p) + np.abs(gw))
        tol = 4 * u * np.abs(p) + 16 * u * np.abs(upd) + 2 * lr * gw_err / (np.sqrt(v64) + eps)
        st_tol = [8 * u * v64 + 4 * (1 - al) * np.abs(gw) * gw_err]
        return p - upd, [v64], tol, st_tol, np.ones(p.shape, bool)
    b1, b2, b3, al, eps = (f(x) for x in (*hp["betas"], hp["alpha"], hp["eps"]))
    c1, c2 = 1 - b1 ** step, math.sqrt(1 - b2 ** step)
    m1 = b1 * state[0] + (1 - b1) * g
    m2 = b3 * state[1] + (1 - b3) * g
    nu = b2 * state[2] + (1 - b2) * g * g
    upd = lr * (m1 / c1 + al * m2) / (np.sqrt(nu) / c2 + eps)
    p64 = (p - upd) * (1 - lr * wd)
    tol = 4 * u * np.abs(p) + 32 * u * np.abs(upd)
    st_tol = [4 * u * (np.abs(b1 * state[0]) + np.abs((1 - b1) * g)), 4 * u * (np.abs(b3 * state[1]) + np.abs((1 - b3) * g)), 8 * u * nu]
    return p64, [m1, m2, nu], tol, st_tol, np.ones(p.shape, bool)


@pytest.mark.parametrize("rule", ["lion", "rmsprop", "ademamix"])
def test_within_float64_bound(rule):
    torch.manual_seed(1)
    n = 50_000
    hp = HP[rule]
    p = torch.nn.Parameter((torch.randn(n) * 0.1).cuda())
    opt = make(rule, [p])
    for step in range(1, 4):
        g = torch.randn(n, device="cuda") * 0.01
        p_prev = p.detach().double().cpu().numpy()
        st_prev = [np.zeros(n)] * (3 if rule == "ademamix" else 1) if step == 1 else [s.astype(np.float64) for s in
                                                                                       gpu_state(rule, opt.state[p])]
        p.grad = g
        opt.step()
        p64, st64, tol, st_tol, sure = _f64_update(rule, p_prev, g.double().cpu().numpy(), st_prev, step, hp)
        got = p.detach().double().cpu().numpy()
        err = np.abs(got - p64)
        assert np.all(err[sure] <= tol[sure]), (step, float((err / tol)[sure].max()))
        assert sure.mean() > 0.999
        assert np.abs(got - p_prev).min() > 0 if rule == "lion" else np.abs(got - p_prev).mean() > 1e3 * tol.mean()  # not vacuous
        for a, b, t in zip(gpu_state(rule, opt.state[p]), st64, st_tol):
            assert np.all(np.abs(a - b) <= t + 1e-30), step


@pytest.mark.parametrize("weight_decay", [0.0, 0.01])
def test_rmsprop_matches_torch(weight_decay):
    import qlora_b200 as q

    torch.manual_seed(2)
    w = torch.randn(256, 65, device="cuda")
    pa, pb = torch.nn.Parameter(w.clone()), torch.nn.Parameter(w.clone())
    oa = q.optim.RMSprop([pa], lr=1e-3, alpha=0.99, eps=1e-8, weight_decay=weight_decay)
    ob = torch.optim.RMSprop([pb], lr=1e-3, alpha=0.99, eps=1e-8, weight_decay=weight_decay, momentum=0, centered=False)
    for _ in range(5):
        g = torch.randn_like(w)
        pa.grad, pb.grad = g.clone(), g.clone()
        oa.step()
        ob.step()
    assert not torch.equal(pa, w)
    assert torch.allclose(pa, pb, rtol=1e-5, atol=1e-7)
    assert torch.allclose(oa.state[pa]["state1"].view_as(w), ob.state[pb]["square_avg"], rtol=1e-5, atol=1e-12)


def test_lion_zero_direction_moves_only_by_decay():
    """c = b1*m + (1-b1)*g = 0 (zero state, zero gradient): sign(c) = 0, so the element moves only by the weight decay."""
    import qlora_b200 as q

    p = torch.nn.Parameter(torch.ones(1000, device="cuda"))
    g = torch.randn(1000, device="cuda")
    g[::3] = 0
    p.grad = g
    lr, wd = 1e-2, 0.1
    q.optim.Lion([p], lr=lr, weight_decay=wd).step()
    decay = np.float32(1) - np.float32(np.float32(lr) * np.float32(wd))
    got = p.detach().cpu().numpy()
    assert np.all(got[::3] == decay)
    moved = np.ones(1000, bool)
    moved[::3] = False
    want = decay - np.float32(lr) * np.sign(g.cpu().numpy()[moved]).astype(np.float32)
    assert np.array_equal(got[moved], want)


@pytest.mark.parametrize("rule", ["lion", "ademamix"])
def test_paged_equals_resident_and_survives_eviction(rule):
    torch.manual_seed(3)
    w = (torch.randn(300, 77, device="cuda") * 0.1).to(torch.bfloat16)
    pr, pp = torch.nn.Parameter(w.clone()), torch.nn.Parameter(w.clone())
    orr, op = make(rule, [pr], paged=False), make(rule, [pp], paged=True)
    for k in range(4):
        g = torch.randn_like(w) * 0.01
        pr.grad, pp.grad = g.clone(), g.clone()
        if k == 3:   # evict the paged state to the host; the next eager step prefetches it back
            for b in op._paged[id(pp)]:
                b.prefetch(False)
            torch.cuda.synchronize()
        orr.step()
        op.step()
        assert torch.equal(pr, pp), k
        for a, b in zip(gpu_state(rule, orr.state[pr]), gpu_state(rule, op.state[pp])):
            assert np.array_equal(a, b) and np.isfinite(b).all(), k
    assert set(op.state[pp]) == ({"step", "state1", "state2"} if rule == "ademamix" else {"step", "state1"})
    assert all(torch.is_tensor(v) for v in op.state[pp].values())


def _flat_views(flat, shapes):
    params, off = [], 0
    for a, b in shapes:
        params.append(torch.nn.Parameter(flat[off:off + a * b].view(a, b)))
        off += a * b
    return params


SHAPES = [(64, 40), (40, 64), (16, 129)]


@pytest.mark.parametrize("rule,paged", RULE_PAGED)
def test_state_dict_resume_bitwise(rule, paged, tmp_path):
    """optimizer.pt as HF Trainer writes it (torch.save -> torch.load(weights_only=True) -> load_state_dict), per parameter
    and after step_flat: the resumed run equals the uninterrupted one bit for bit."""
    torch.manual_seed(4)
    w = (torch.randn(300, 33, device="cuda") * 0.1).to(torch.bfloat16)
    grads = [torch.randn_like(w) * 0.01 for _ in range(4)]

    def per_param(p, opt, gs):
        for g in gs:
            p.grad = g.clone()
            opt.step()

    pa = torch.nn.Parameter(w.clone())
    per_param(pa, make(rule, [pa], paged), grads)
    pb = torch.nn.Parameter(w.clone())
    ob = make(rule, [pb], paged)
    per_param(pb, ob, grads[:2])
    f = tmp_path / "optimizer.pt"
    torch.save(ob.state_dict(), f)
    pc = torch.nn.Parameter(pb.detach().clone())
    del ob
    oc = make(rule, [pc], paged)
    oc.load_state_dict(torch.load(f, weights_only=True))
    if paged:
        assert oc.state[pc]["state1"].data_ptr() == oc._paged[id(pc)][0].ptr
    per_param(pc, oc, grads[2:])
    assert torch.equal(pc, pa) and float(oc.state[pc]["step"]) == 4

    # step_flat, parameters listed in another order than the flat buffer holds them
    n = sum(a * b for a, b in SHAPES)
    wf = (torch.randn(n, device="cuda") * 0.05).to(torch.bfloat16)
    fgrads = [(torch.randn(n, device="cuda") * 0.01).to(torch.bfloat16) for _ in range(4)]
    scales = [1.0, 0.5, 0.25, 1.0]

    def run(flat_p, opt, steps):
        flat_g = torch.empty_like(flat_p)
        scale = torch.ones((), device="cuda")
        for g, sc in steps:
            flat_g.copy_(g)
            scale.fill_(sc)
            opt.step_flat(flat_p, flat_g, grad_scale=scale)

    flat_a = wf.clone()
    run(flat_a, make(rule, _flat_views(flat_a, SHAPES)[::-1], paged, capturable=True), list(zip(fgrads, scales)))
    flat_b = wf.clone()
    ob = make(rule, _flat_views(flat_b, SHAPES)[::-1], paged, capturable=True)
    run(flat_b, ob, list(zip(fgrads, scales))[:2])
    sd = ob.state_dict()
    assert sorted(sd["state"]) == [0, 1, 2] and all(float(st["step"]) == 2 for st in sd["state"].values())
    if rule == "ademamix":   # the [2, numel_p] slice of the flat [2, N] buffer
        assert all(st["state1"].shape == (2, p.numel()) for st, p in zip(sd["state"].values(), ob.param_groups[0]["params"]))
    torch.save(sd, f)
    flat_c = flat_b.clone()
    del ob, sd
    oc = make(rule, _flat_views(flat_c, SHAPES)[::-1], paged, capturable=True)
    oc.load_state_dict(torch.load(f, weights_only=True))
    run(flat_c, oc, list(zip(fgrads, scales))[2:])
    assert torch.equal(flat_c, flat_a)
    assert float(oc._step_dev.item()) == 4
    if paged:
        assert oc._paged[id(oc._flat_key)][0].ptr == oc._flat[0].data_ptr()


@pytest.mark.parametrize("rule", ["lion", "rmsprop", "ademamix"])
def test_captured_step_with_varying_grad_scale_equals_eager(rule):
    torch.manual_seed(5)
    w = (torch.randn(4096, 17, device="cuda") * 0.1).to(torch.bfloat16)
    grads = [torch.randn_like(w) * 0.02 for _ in range(5)]
    scales = [1.0, 0.5, 0.25, 1.0, 0.125]
    kw = dict(t_alpha=3, t_beta3=3) if rule == "ademamix" else {}
    pe = torch.nn.Parameter(w.clone())
    oe = make(rule, [pe], **kw)
    for g, sc in zip(grads, scales):
        pe.grad = (g.float() * sc).to(torch.bfloat16)   # power-of-two scales: exact in bf16
        oe.step()
    pg = torch.nn.Parameter(w.clone())
    og = make(rule, [pg], capturable=True, **kw)
    static_g = torch.zeros_like(w)
    scale_dev = torch.ones((), device="cuda", dtype=torch.float32)
    pg.grad = static_g
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):     # warm-up step outside the graph (allocates the state), then rewind it
        og.step(grad_scale=scale_dev)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    with torch.no_grad():
        pg.copy_(w)
    for k in ("state1", "state2"):
        if k in og.state[pg]:
            og.state[pg][k].zero_()
    og._step_dev.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        og.step(grad_scale=scale_dev)
    for g, sc in zip(grads, scales):
        static_g.copy_(g)
        scale_dev.fill_(sc)
        graph.replay()
    torch.cuda.synchronize()
    assert float(og._step_dev.item()) == 5
    assert not torch.equal(pg, w)
    assert torch.equal(pg, pe)
    for a, b in zip(gpu_state(rule, og.state[pg]), gpu_state(rule, oe.state[pe])):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("rule,paged", RULE_PAGED)
def test_step_flat_equals_per_parameter_steps(rule, paged):
    torch.manual_seed(6)
    n = sum(a * b for a, b in SHAPES)
    flat_p = (torch.randn(n, device="cuda") * 0.1).to(torch.bfloat16)
    flat_g = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    params = _flat_views(flat_p, SHAPES)
    ref_params = [torch.nn.Parameter(p.detach().clone()) for p in params]
    opt = make(rule, params, paged, capturable=True)
    ref = make(rule, ref_params)
    scale = torch.ones((), device="cuda")
    for step, sc in enumerate([1.0, 0.5, 0.25]):
        flat_g.copy_((torch.randn(n, device="cuda") * 0.02).to(torch.bfloat16))
        scale.fill_(sc)
        off = 0
        for rp, (a, b) in zip(ref_params, SHAPES):
            rp.grad = (flat_g[off:off + a * b].float() * sc).to(torch.bfloat16).view(a, b).clone()
            off += a * b
        opt.step_flat(flat_p, flat_g, grad_scale=scale)
        ref.step()
        for p, rp in zip(params, ref_params):
            assert torch.equal(p, rp), step
    assert float(opt._step_dev.item()) == 3
    sd = opt.state_dict()["state"]
    for i, rp in enumerate(ref_params):
        for k in ref.state[rp]:
            if k != "step":
                assert torch.equal(sd[i][k], ref.state[rp][k]), (i, k)


# ---- the benchmarked training step (tests/test_gpu_bench_step.py's BenchStep) with Lion and AdEMAMix ----------------------

BENCH_RULES = {"PagedLion32bit": dict(lr=LR, betas=(0.9, 0.99), weight_decay=0.0),
               "PagedAdEMAMix32bit": dict(lr=LR, betas=(0.9, 0.999, 0.9999), alpha=5.0, eps=1e-8, weight_decay=0.0)}


def _bench_step(H, cfg, name):
    import qlora_b200 as q

    bs = BenchStep(H, cfg)
    bs.opt = getattr(q.optim, name)(bs.model.trainable_parameters(), capturable=True, **BENCH_RULES[name])
    return bs


def _f64_bench_update(name, gs, clips):
    """The update of the last of len(gs) steps from zero state, in float64 with the fp32 hyper-parameters (weight decay 0),
    and whether its direction is decided beyond fp32 rounding (Lion's sign)."""
    hp = {k: (tuple(float(np.float32(b)) for b in v) if k == "betas" else float(np.float32(v))) for k, v in BENCH_RULES[name].items()}
    lr = hp["lr"]
    if name == "PagedLion32bit":
        b1, b2 = hp["betas"]
        m = 0.0
        for g, c in zip(gs[:-1], clips[:-1]):
            m = b2 * m + (1 - b2) * c * g
        d = b1 * m + (1 - b1) * clips[-1] * gs[-1]
        scale = np.abs(b1 * m) + np.abs((1 - b1) * clips[-1] * gs[-1])
        return -lr * np.sign(d), (np.abs(d) > 2.0 ** -20 * scale) | (d == 0)
    b1, b2, b3 = hp["betas"]
    m1 = m2 = nu = 0.0
    for g, c in zip(gs, clips):
        gi = c * g
        m1 = b1 * m1 + (1 - b1) * gi
        m2 = b3 * m2 + (1 - b3) * gi
        nu = b2 * nu + (1 - b2) * gi * gi
    t = len(gs)
    c1, c2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
    return -lr * (m1 / c1 + hp["alpha"] * m2) / (np.sqrt(nu) / c2 + hp["eps"]), np.ones(np.shape(m1), bool)


def _bf16(x):
    return torch.from_numpy(x).to(torch.bfloat16).double().numpy()


@pytest.mark.parametrize("name", sorted(BENCH_RULES))
def test_bench_step_update_matches_float64(H, deterministic, monkeypatch, name):
    """Every adapter weight after each of two steps is the bf16 rounding of the float64 update computed from the step's own
    gradient and clip coefficient."""
    with monkeypatch.context() as mp:
        _bench_settings(mp, H, fused=True)
        bs = _bench_step(H, CASES["fused_p0.1_accum2"], name)
        p_prev = bs.gsync.flat_param.double().cpu().numpy()
        steps = [bs.step(0), bs.step(1)]
    gs = [s["grad"].double().cpu().numpy() for s in steps]
    clips = [float(s["clip"]) for s in steps]
    for k, s in enumerate(steps):
        p_new = s["params"].double().cpu().numpy()
        upd, sure = _f64_bench_update(name, gs[:k + 1], clips[:k + 1])
        want = p_prev + upd
        tol = 2.0 ** -20 * np.abs(p_prev) + 2.0 ** -18 * np.abs(upd)
        ok = (p_new >= _bf16(want - tol)) & (p_new <= _bf16(want + tol))
        bad = np.flatnonzero(~ok & sure)[:4]
        assert (ok | ~sure).all() and sure.mean() > 0.999, (k, int((~ok & sure).sum()), bad, p_prev[bad], upd[bad], p_new[bad])
        assert (p_new != p_prev).mean() > 0.5, k
        p_prev = p_new


@pytest.mark.parametrize("name", sorted(BENCH_RULES))
def test_bench_step_graph_replay_equals_eager(H, deterministic, monkeypatch, name):
    """One graph per micro-step kind, replayed for two optimizer steps from a restored state, equals eager bit for bit."""
    with monkeypatch.context() as mp:
        _bench_settings(mp, H, fused=True)
        bs = _bench_step(H, CASES["fused_p0.1_accum2"], name)
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
