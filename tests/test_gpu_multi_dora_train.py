"""Training several DoRA adapters over one NF4 base in one batch (`dora_linear4bit_group_multi`, DESIGN.md §6e).

Norms.  n_a = ||W + s B_a A_a||_row from the kernels (one fused forward P = A_stack . W^T with a bf16-rounded fp32 output,
the Gram matrices and the per-row expansion) against float64 norms of the C oracle's weights.  §6b's argument: P is rounded
to the compute dtype (relative 2^-9 per entry), so the cross term is off by at most 2^-9 . 2s . sum_j |B P| and n^2 by less
than 2^-8 of itself unless the adapter is as large as W and aligned against it; the fp32 sums add ~1e-6.  Bound: 2^-8 per
row, relative.

Outputs and gradients.  The float64 restatement takes c and n from the kernels (so norm error is not counted twice) and
rounds where the definition rounds: the base outputs rn(x . W^T) and rn(xd . W^T), U, y, Q (dropout), dQ, dD, G, dx (twice:
the base dX launch, then the adapter term) and dxd (twice).  dm is checked against sum_t dY . Q / n with Q the pre-scale
term as the path keeps it: y / c without dropout (the output rounded once, then divided: the path's stated choice), the
rounded Q with it.  What is left is the fp32 summation order of the kernels against float64, which moves an element by one
ulp only where it lands on the other side of a rounding boundary: as tests/test_gpu_multi_adapter_train.py argues, a
Frobenius-relative error of at most 2^-8 sqrt(f) for a share f of flipped elements, so TOL = 1e-3 with every element
within 1.01 ulp of max|ref|.  The same exceptions apply for the same reasons: dA, dB and dm under bf16 contract operands
(G, U, dQ, the rounded y) that differ by one ulp where a flip occurred, with few rows per adapter (2.5e-3, the segmented
path's bf16 bar), and outputs at 1 to 16 rows, where one ulp moves on a single row are not averaged (4e-3).  y rounds twice
(the base output, then the scaled sum), so a one-ulp flip of the base output reaches the second rounding multiplied by c
(or c - 1 with dropout): its elements are held to 1 + max c ulp instead of 1.
Negative controls (two adapters' magnitudes swapped, c dropped) must exceed these bounds by far.
"""
import os
import subprocess
import sys

import pytest
import torch

from fp16_helpers import oracle_w16
from gpu_helpers import make_act, make_weight, max_err_ulps, oracle_weight, rel_err

pytestmark = pytest.mark.gpu

BF16, H16 = torch.bfloat16, torch.float16
RANKS = [8, 16, 72, 256]
TOL, TOL_BF16_WGRAD, TOL_FEW_ROWS = 1e-3, 2.5e-3, 4e-3
SHAPES = {"qkv": (4096, 4096, 3), "gate_up": (11008, 4096, 2), "down": (4096, 11008, 1), "ragged": (1000, 1088, 2)}
CDTS = {"bf16": (BF16, BF16), "fp16": (H16, H16), "bf16_over_fp16_state": (BF16, H16)}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _q():
    import qlora_b200 as q

    return q


def _base(n, k, cdt, sdt, seed):
    q = _q()
    lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=cdt, quant_type="nf4")
    lin.weight = q.nn.Params4bit(make_weight(n, k, seed=seed, dtype=sdt), requires_grad=False, compress_statistics=True,
                                 quant_type="nf4", module=lin)
    return lin.cuda()


def _w64(base, c_oracle, cdt, sdt):
    w = base.weight
    if sdt == BF16:
        return torch.from_numpy(oracle_weight(w.data, w.quant_state, c_oracle)).cuda().double()
    return torch.from_numpy(oracle_w16(c_oracle, w.data, w.quant_state)).cuda().to(cdt).double()


def _adapters(n, k, na, cdt, seed, ranks=RANKS):
    """{name: (A, B, magnitude, scaling)}, leaves that require grad; the magnitude is near the norm of W + s B A (peft's
    initialisation, ||W_f|| ~ 0.02 sqrt(K)) with a spread, so c stays near 1 but not at it."""
    out = {}
    for i in range(na):
        r = ranks[i % len(ranks)]
        a = make_weight(r, k, seed=seed + 3 * i, dtype=cdt, scale=k ** -0.5).requires_grad_()
        b = make_weight(n, r, seed=seed + 3 * i + 1, dtype=cdt, scale=0.05).requires_grad_()
        g = torch.Generator(device="cpu").manual_seed(seed + 3 * i + 2)
        m = (0.02 * k ** 0.5 * (1.0 + 0.2 * torch.rand(n, generator=g))).to(cdt).cuda().requires_grad_()
        out[f"ad{i}"] = (a, b, m, 0.5 + 0.25 * (i % 3))
    return out


def _rows(m, na, seed=0):
    """Every third row a base row (alternately -1 and an index past the set), the others spread over the adapters."""
    return torch.tensor([(-1 if t % 2 else na + 3) if t % 3 == 1 else (7 * t + seed) % na for t in range(m)], dtype=torch.int32,
                        device="cuda")


def _setup(group, cdt_name, na, seed=0, ranks=RANKS):
    n, k, p = SHAPES[group]
    cdt, sdt = CDTS[cdt_name]
    bases = [_base(n, k, cdt, sdt, seed=31 * i + seed + 1) for i in range(p)]
    adapters = [_adapters(n, k, na, cdt, seed=1000 * (i + 1) + seed, ranks=ranks) for i in range(p)]
    sets = [_q().DoraAdapterSet(a) for a in adapters]
    return bases, adapters, sets, cdt, sdt


def _kernel_norms(bases, sets):
    """(c, n) [P, n_adapters, N] as the forward computes them."""
    from qlora_b200 import _ops
    from qlora_b200 import functional as F

    states = [b.weight.quant_state for b in bases]
    packeds = [b.weight.t() for b in bases]
    sts = [F._state_tensors(qs, packeds[0].device) for qs in states]
    s0 = sets[0]
    n_out, k_in = states[0].shape
    return _ops.dora_segmented_norm([s.table for s in sets], [s.mag_table for s in sets], s0.stack_rows, s0.rank_offsets,
                                    s0.gram_offsets, s0.rank_total, s0.gram_total, packeds,
                                    [a_f32 if a_u8 is None else a_u8 for a_u8, _, _, _, a_f32 in sts], [t[1] for t in sts],
                                    [t[2] for t in sts], [t[3] for t in sts], n_out, k_in, states[0].dtype,
                                    [F.weight_row_norm2(p, qs) for p, qs in zip(packeds, states)], s0.dtype, len(s0),
                                    max(s.rmax for s in sets))


def _check(got, want, what, tol=TOL, ulps=1.01):
    g, w = got.detach().float().cpu().numpy(), want.float().cpu().numpy()
    e, u = rel_err(g, w), max_err_ulps(g, w)
    assert e <= tol and u <= ulps, f"{what}: rel_F={e:.3e}, max err {u:.2f} ulp of max|ref|"
    return e


def _reference(x, xls, dys, w64s, adapters, rows, cs, nrms, cdt, swap_mag=None, drop_c=False):
    """float64 (ys, dx, dxds, {(p, name): (dA, dB, dm)}) with c and n from the kernels.  `swap_mag` = (a, b) gives adapter
    a's rows adapter b's magnitude scale, `drop_c` takes c = 1 (plain LoRA): the negative controls."""
    rn = lambda t: t.to(cdt).double()  # noqa: E731
    x64 = x.double()
    names = list(adapters[0])
    split = xls is not None
    dq_all, dd_all, ys, grads = [], [], [], {}
    lora_dx = torch.zeros_like(x64)
    dxds = []
    for p, (ad, dy, w64) in enumerate(zip(adapters, dys, w64s)):
        xl = xls[p].double() if split else x64
        dy64 = dy.double()
        ybase = rn(x64 @ w64.t())
        qb = rn(xl @ w64.t()) if split else None
        y, dq = ybase.clone(), dy64.clone()
        dd = torch.zeros_like(dy64)
        dxd = torch.zeros_like(x64)
        for i, name in enumerate(names):
            a, b, _, s = (t.detach().double() if torch.is_tensor(t) else t for t in ad[name])
            sel = (rows.long() == i).nonzero().flatten()
            j = i if swap_mag is None or i != swap_mag[0] else swap_mag[1]
            c = torch.ones_like(cs[p, j].double()) if drop_c else cs[p, j].double()
            nrm = nrms[p, i].double()
            if not sel.numel():
                grads[(p, name)] = (torch.zeros_like(a), torch.zeros_like(b), torch.zeros_like(nrm))
                continue
            u = rn(s * (xl[sel] @ a.t()))
            ub = u @ b.t()
            if split:
                y[sel] = rn(ybase[sel] + (c - 1) * qb[sel] + c * ub)
                qq = rn(qb[sel] + ub)
                dd[sel] = rn(dy64[sel] * (c - 1))
            else:
                y[sel] = rn(c * (ybase[sel] + ub))
                qq = y[sel] / c
            dq[sel] = rn(dy64[sel] * c)
            g = rn(s * (dq[sel] @ b))
            if split:
                dxd[sel] = g @ a
            else:
                lora_dx[sel] += g @ a
            grads[(p, name)] = (g.t() @ xl[sel], dq[sel].t() @ u, (dy64[sel] * qq).sum(0) / nrm)
        if split:
            dxd = rn(rn(dd @ w64) + dxd)
        ys.append(y)
        dq_all.append(dq)
        dxds.append(dxd)
    if split:
        dx = rn(sum(d.double() @ w for d, w in zip(dys, w64s)))
    else:
        dx = rn(rn(sum(d @ w for d, w in zip(dq_all, w64s))) + lora_dx)
    return ys, dx, dxds, grads


def _run(x, bases, sets, rows, dys, x_loras=None):
    q = _q()
    x = x.detach().requires_grad_()
    xls = None if x_loras is None else [t.detach().requires_grad_() for t in x_loras]
    params = [t for s in sets for t in s.lora_as + s.lora_bs + s.magnitudes]
    for t in params:
        t.grad = None
    ys = q.dora_linear4bit_group_multi(x, bases, sets, rows, xls)
    torch.autograd.backward(list(ys), list(dys))
    return ys, x.grad, None if xls is None else [t.grad for t in xls]


def _grads(sets):
    return {(p, name): (s.lora_as[i].grad, s.lora_bs[i].grad, s.magnitudes[i].grad)
            for p, s in enumerate(sets) for i, name in enumerate(s.names)}


CASES = ([(g, "bf16", d, m) for g in SHAPES for d in (False, True) for m in (12, 700)]
         + [(g, c, d, m) for g in ("qkv", "ragged") for c in ("fp16", "bf16_over_fp16_state") for d in (False, True)
            for m in (12, 700)])


@pytest.mark.parametrize("group,cdt_name,dropout,m", CASES)
def test_outputs_and_gradients_against_float64(c_oracle, group, cdt_name, dropout, m):
    na = 4 if m < 100 else 16
    bases, adapters, sets, cdt, sdt = _setup(group, cdt_name, na, seed=m)
    n, k, p = SHAPES[group]
    x = make_act(m, k, seed=5 + m).to(cdt)
    xls = [torch.nn.functional.dropout(x.float(), 0.1).to(cdt) for _ in range(p)] if dropout else None
    rows = _rows(m, na)
    dys = [(make_act(m, n, seed=70 + i) * 0.1).to(cdt) for i in range(p)]
    cs, nrms = _kernel_norms(bases, sets)
    ys, dx, dxls = _run(x, bases, sets, rows, dys, xls)
    w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
    ry, rdx, rdxds, rgrads = _reference(x, xls, dys, w64s, adapters, rows, cs, nrms, cdt)
    tol_y = TOL_FEW_ROWS if m <= 16 else TOL
    tol_w = TOL_BF16_WGRAD if cdt == BF16 else TOL
    # y rounds twice, and a one-ulp flip of the base output reaches the second rounding scaled by c (or c - 1): 1 + max c ulp
    for i in range(p):
        _check(ys[i], ry[i], f"y[{i}]", tol_y, ulps=1.01 + float(cs[i].abs().max()))
    _check(dx, rdx, "dx")
    if dropout:
        for i in range(p):
            _check(dxls[i], rdxds[i], f"dxd[{i}]")
    got = _grads(sets)
    da = torch.cat([got[key][0].flatten() for key in rgrads])
    db = torch.cat([got[key][1].flatten() for key in rgrads])
    dm = torch.cat([got[key][2].flatten() for key in rgrads])
    _check(da, torch.cat([v[0].flatten() for v in rgrads.values()]), "dA", tol_w)
    _check(db, torch.cat([v[1].flatten() for v in rgrads.values()]), "dB", tol_w)
    _check(dm, torch.cat([v[2].flatten() for v in rgrads.values()]), "dm", tol_w)
    if group == "qkv" and m > 16:
        # negative controls: two adapters' magnitude scales swapped, or c dropped, exceed the bars by far
        for kw in (dict(swap_mag=(0, 1)), dict(drop_c=True)):
            bad_y = _reference(x, xls, dys, w64s, adapters, rows, cs, nrms, cdt, **kw)[0]
            e = rel_err(ys[0].detach().float().cpu().numpy(), bad_y[0].float().cpu().numpy())
            assert e > 3 * tol_y, (kw, e)


@pytest.mark.parametrize("na", [1, 4, 64, 2048])
def test_norms_against_float64(c_oracle, na):
    """Every adapter's norm of the 7B q/k/v shapes at mixed ranks 8..256 (8 and 16 at 2048 adapters), within 2^-8 per row of
    a float64 norm of the oracle's weight; at most 12 adapters per problem are restated in float64."""
    ranks = [8, 16] if na > 64 else [8, 256, 72, 16, 136]
    bases, adapters, sets, cdt, sdt = _setup("qkv", "bf16", na, seed=na, ranks=ranks)
    cs, nrms = _kernel_norms(bases, sets)
    assert torch.isfinite(cs).all() and (nrms > 0).all()
    names = sets[0].names
    pick = sorted(set([0, na - 1] + list(range(0, na, max(1, na // 10)))))[:12]
    for p, (base, ad) in enumerate(zip(bases, adapters)):
        w64 = _w64(base, c_oracle, cdt, sdt)
        for i in pick:
            a, b, mg, s = ad[names[i]]
            ref = torch.linalg.norm(w64 + s * (b.detach().double() @ a.detach().double()), dim=1)
            err = ((nrms[p, i].double() - ref).abs() / ref).max().item()
            assert err <= 2.0 ** -8, (p, i, err)
            assert torch.allclose(cs[p, i].double(), mg.detach().double() / nrms[p, i].double(), rtol=1e-6, atol=0)


def test_agrees_with_single_adapter_paths():
    """Every row on one adapter, bf16 over a bf16 state: the same step through `dora_linear4bit_group` (row-scaled fused
    launches, one rounding) and `dora_linear4bit_peft` (forward).  Each is within its own bound of float64, so they agree to
    the sum of those bounds plus the different roundings of the paths (one against two): 5e-3 for y and dx, 1e-2 for the
    adapter gradients, which contract the rounded operands."""
    q = _q()
    bases, adapters, sets, cdt, _ = _setup("qkv", "bf16", 1, seed=3, ranks=[64])
    m = 512
    x = make_act(m, 4096, seed=11)
    dys = [(make_act(m, 4096, seed=80 + i) * 0.1) for i in range(3)]
    rows = torch.zeros(m, dtype=torch.int32, device="cuda")
    ys, dx, _ = _run(x, bases, sets, rows, dys)
    got = _grads(sets)
    xr = x.detach().requires_grad_()
    ads = [a["ad0"] for a in adapters]
    leaves = [(a.detach().clone().requires_grad_(), b.detach().clone().requires_grad_(), mg.detach().clone().requires_grad_())
              for a, b, mg, _ in ads]
    ref = q.dora_linear4bit_group(xr, bases, [t[0] for t in leaves], [t[1] for t in leaves], [t[2] for t in leaves], ads[0][3])
    torch.autograd.backward(list(ref), dys)
    for i in range(3):
        assert rel_err(ys[i].detach().float().cpu().numpy(), ref[i].detach().float().cpu().numpy()) <= 5e-3
        for j, g in enumerate(got[(i, "ad0")]):
            assert rel_err(g.float().cpu().numpy(), leaves[i][j].grad.float().cpu().numpy()) <= 1e-2, (i, j)
        with torch.no_grad():
            peft = q.dora_linear4bit_peft(x, bases[i], *[t.detach() for t in ads[i][:3]], ads[i][3])
        assert rel_err(ys[i].detach().float().cpu().numpy(), peft.float().cpu().numpy()) <= 5e-3
    assert rel_err(dx.float().cpu().numpy(), xr.grad.float().cpu().numpy()) <= 5e-3


@pytest.mark.parametrize("dropout", [False, True])
def test_base_rows_and_empty_adapters(dropout):
    """Base and out-of-range rows return Linear4bit's bits, and their dx the base dX launch's; adapters without rows get
    exact zeros for dA, dB and dm."""
    bases, adapters, sets, cdt, _ = _setup("down", "bf16", 6, seed=21)
    m = 300
    x = make_act(m, 11008, seed=2)
    rows = torch.tensor([[-1, 0, 9, 2][t % 4] for t in range(m)], dtype=torch.int32, device="cuda")   # adapters 1, 3-5 empty
    dys = [make_act(m, 4096, seed=3) * 0.1]
    xls = [torch.nn.functional.dropout(x.float(), 0.1).to(cdt)] if dropout else None
    ys, dx, dxls = _run(x, bases, sets, rows, dys, xls)
    base_rows = ((rows < 0) | (rows >= 6)).nonzero().flatten()
    xb = x.detach().requires_grad_()
    yb = bases[0](xb)                                         # the same M, so the same kernel schedule
    yb.backward(dys[0])
    assert torch.equal(ys[0].detach()[base_rows], yb.detach()[base_rows])
    assert torch.equal(dx[base_rows], xb.grad[base_rows])
    if dropout:                                               # dx is the base dX launch on every row
        assert torch.equal(dx, xb.grad)
    if dropout:
        assert (dxls[0][base_rows] == 0).all()
    got = _grads(sets)
    for name in ("ad1", "ad3", "ad4", "ad5"):
        for g in got[(0, name)]:
            assert (g == 0).all() and not torch.signbit(g).any(), name
    for name in ("ad0", "ad2"):
        assert all(g.abs().sum() > 0 for g in got[(0, name)]), name


def test_determinism_no_sync_and_checkpoint():
    bases, adapters, sets, cdt, _ = _setup("gate_up", "bf16", 8, seed=4)
    m = 700
    x = make_act(m, 4096, seed=9)
    rows = _rows(m, 8)
    dys = [make_act(m, 11008, seed=10 + i) * 0.1 for i in range(2)]
    runs = []
    for _ in range(2):
        ys, dx, _ = _run(x, bases, sets, rows, dys)
        runs.append(([y.detach().clone() for y in ys], dx.clone(), {k: tuple(t.clone() for t in v) for k, v in _grads(sets).items()}))
    (y0, dx0, g0), (y1, dx1, g1) = runs
    assert all(torch.equal(a, b) for a, b in zip(y0, y1)) and torch.equal(dx0, dx1)
    assert all(torch.equal(a, b) for k in g0 for a, b in zip(g0[k], g1[k]))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(x, bases, sets, rows, dys)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    # a checkpointed step (forward recomputed in the backward) gives the plain step's bits
    import qlora_b200 as q
    from torch.utils.checkpoint import checkpoint

    xc = x.detach().requires_grad_()
    for s in sets:
        for t in s.lora_as + s.lora_bs + s.magnitudes:
            t.grad = None
    ys = checkpoint(lambda t: q.dora_linear4bit_group_multi(t, bases, sets, rows), xc, use_reentrant=False)
    torch.autograd.backward(list(ys), dys)
    assert all(torch.equal(a.detach(), b) for a, b in zip(ys, y0)) and torch.equal(xc.grad, dx0)
    g2 = _grads(sets)
    assert all(torch.equal(a, b) for k in g0 for a, b in zip(g0[k], g2[k]))


def test_cuda_graph_replay_after_rewriting_rows():
    import qlora_b200 as q

    bases, adapters, sets, cdt, _ = _setup("qkv", "bf16", 5, seed=6)
    m = 640
    x = make_act(m, 4096, seed=1).requires_grad_()
    dys = [make_act(m, 4096, seed=2 + i) * 0.1 for i in range(3)]
    rows = _rows(m, 5).clone()
    params = [t for s in sets for t in s.lora_as + s.lora_bs + s.magnitudes]

    def step():
        ys = q.dora_linear4bit_group_multi(x, bases, sets, rows)
        grads = torch.autograd.grad(list(ys), [x] + params, dys)
        return [y.detach() for y in ys] + list(grads)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step()
    rows.copy_(_rows(m, 5, seed=3))
    g.replay()
    torch.cuda.synchronize()
    eager = step()
    assert all(torch.equal(a, b) for a, b in zip(outs, eager))


def test_reads_stay_inside_nan_padded_operands():
    """Adapters, magnitudes and activations cut out of NaN-filled buffers: a read past any of them would make a result NaN."""
    q = _q()
    cdt = BF16
    n, k = 1000, 1088
    bases = [_base(n, k, cdt, cdt, seed=40 + i) for i in range(2)]

    def padded(t):
        buf = torch.full((t.numel() + 4096,), float("nan"), dtype=t.dtype, device="cuda")
        view = buf[2048:2048 + t.numel()].view(t.shape)
        view.copy_(t)
        return view.requires_grad_()

    sets = []
    for p in range(2):
        ad = _adapters(n, k, 5, cdt, seed=300 + p, ranks=[8, 256, 72])
        sets.append(q.DoraAdapterSet({name: (padded(a.detach()), padded(b.detach()), padded(mg.detach()), s)
                                      for name, (a, b, mg, s) in ad.items()}))
    m = 333
    xbuf = torch.full((m + 2, k + 64), float("nan"), dtype=cdt, device="cuda")
    x = xbuf[1:m + 1, :k]
    x.copy_(make_act(m, k, seed=8))
    dys = [make_act(m, n, seed=9 + i) * 0.1 for i in range(2)]
    xls = [torch.nn.functional.dropout(x.float(), 0.1).to(cdt) for _ in range(2)]
    for xl in (None, xls):
        ys, dx, dxls = _run(x, bases, sets, _rows(m, 5), dys, xl)
        assert all(torch.isfinite(y).all() for y in ys) and torch.isfinite(dx).all()
        assert all(torch.isfinite(t).all() for v in _grads(sets).values() for t in v)


def test_adamw_step_moves_only_the_jobs_adapters():
    """Two jobs in one batch (adapters 0 and 2 of three): one AdamW step changes their A, B and magnitude and leaves
    adapter 1, which no row uses, exactly as it was."""
    bases, adapters, sets, cdt, _ = _setup("ragged", "bf16", 3, seed=12)
    m = 256
    x = make_act(m, 1088, seed=4)
    rows = torch.tensor([0 if t < m // 2 else 2 for t in range(m)], dtype=torch.int32, device="cuda")
    dys = [make_act(m, 1000, seed=5 + i) * 0.1 for i in range(2)]
    params = [t for s in sets for t in s.lora_as + s.lora_bs + s.magnitudes]
    before = [t.detach().clone() for t in params]
    opt = torch.optim.AdamW(params, lr=1e-2, weight_decay=0.0)   # a step above one bf16 ulp of m
    _run(x, bases, sets, rows, dys)
    opt.step()
    for s in sets:
        for i in range(3):
            for t in (s.lora_as[i], s.lora_bs[i], s.magnitudes[i]):
                j = next(idx for idx, pp in enumerate(params) if pp is t)
                moved = not torch.equal(t.detach(), before[j])
                assert moved == (i != 1), (i, moved)


def test_fullgraph_compile_in_subprocess():
    env = dict(os.environ)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "multi_dora_compile_case.py")], capture_output=True, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    import json

    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["graph_breaks"] == 0 and all(res["equal"]), res
