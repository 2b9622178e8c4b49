"""Training several LoRA adapters over one NF4 base in one batch (`lora_linear4bit_group_multi`, DESIGN.md §6d): the
segmented forward of the mixed-adapter path and its backward (qlora_b200/csrc/lora_segmented.cu).

Bounds.  Every reference is a float64 restatement on the compute-dtype operands (the C oracle's weights, the adapters, x,
dY) that rounds where the definition rounds: U and G once, dX as rn(rn(sum_p dY_p . W_p) + sum_p G_p . A_p), dA, dB and
dxl once.  The kernels sum in fp32 in another order, so a result differs from the reference only where the fp32 sum lands
on the other side of a rounding boundary than the float64 sum: one ulp on a small share of the elements.  One ulp is at
most 2^-8 (bf16) or 2^-11 (fp16) of an element, so if at most a fraction f of the elements flip, the Frobenius-relative
error is at most 2^-8 sqrt(f) (bf16): 1e-3 allows f up to 6.5 %.  The sums here run over at most 11008 terms of magnitude
O(1) with fp32 unit roundoff 2^-24, about 1e-5 relative, against a rounding spacing of 4e-3 (bf16): flips are well under
1 % of the elements.  So: TOL = 1e-3 for every tensor and compute dtype, and each element within 1.01 ulp of max|ref|.

Two exceptions, both in bf16.  dA and dB (TOL_WGRAD_BF16 = 2.5e-3): they contract G or U, which the reference rounds from
float64 and the kernels from fp32, so the operands themselves differ by one ulp where a flip occurred, and with a few rows
per adapter (64 adapters over 700 rows) a flipped element of G is a sizeable share of its dA row: 1.05e-3 to 1.51e-3 was
measured on an H100 at 64 adapters, every element still within one ulp; 2.5e-3 is the segmented forward's bf16 bound
(tests/test_gpu_mixed_segmented.py).  The forward at 1 to 16 rows (4e-3): y is rounded twice, and over a single row of 4096
elements the share of elements the second rounding moves by one ulp is not averaged over many rows; each element still
within one ulp, and one ulp is at most 2^-7 of an element, so 4e-3 is about half of the elements moved by a full ulp.
"""
import pytest
import torch

from fp16_helpers import oracle_w16
from gpu_helpers import make_act, make_weight, max_err_ulps, oracle_weight, rel_err

pytestmark = pytest.mark.gpu

BF16, H16 = torch.bfloat16, torch.float16
RANKS = [8, 16, 72, 256]
TOL = 1e-3
TOL_WGRAD_BF16 = 2.5e-3
SHAPES = {"qkv": (4096, 4096, 3), "gate_up": (11008, 4096, 2), "down": (4096, 11008, 1), "ragged": (1000, 1088, 2)}
CDTS = {"bf16": (BF16, BF16), "fp16": (H16, H16), "bf16_over_fp16_state": (BF16, H16)}


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
    """{name: (A, B, scaling)} with A and B leaf tensors that require grad; adapter i has rank ranks[i % len(ranks)] and the
    same scaling in every problem of a group."""
    out = {}
    for i in range(na):
        r = ranks[i % len(ranks)]
        a = make_weight(r, k, seed=seed + 2 * i, dtype=cdt, scale=k ** -0.5).requires_grad_()
        b = make_weight(n, r, seed=seed + 2 * i + 1, dtype=cdt, scale=0.05).requires_grad_()
        out[f"ad{i}"] = (a, b, 0.5 + 0.25 * (i % 3))
    return out


def _rows(m, na, seed=0):
    """Row indices: every third row a base row, the others spread over the adapters (some adapters may get no row)."""
    return torch.tensor([-1 if t % 3 == 1 else (7 * t + seed) % na for t in range(m)], dtype=torch.int32, device="cuda")


def _setup(group, cdt_name, na, seed=0, ranks=RANKS):
    n, k, p = SHAPES[group]
    cdt, sdt = CDTS[cdt_name]
    bases = [_base(n, k, cdt, sdt, seed=31 * i + seed + 1) for i in range(p)]
    adapters = [_adapters(n, k, na, cdt, seed=1000 * (i + 1) + seed, ranks=ranks) for i in range(p)]
    sets = [_q().LoraAdapterSet(a) for a in adapters]
    return bases, adapters, sets, cdt, sdt


def _check(got, want, what, tol=TOL, ulps=1.01):
    g, w = got.detach().float().cpu().numpy(), want.float().cpu().numpy()
    e, u = rel_err(g, w), max_err_ulps(g, w)
    assert e <= tol and u <= ulps, f"{what}: rel_F={e:.3e}, max err {u:.2f} ulp of max|ref|"
    return e


def _reference(x, xls, dys, w64s, adapters, rows, cdt, drop_problem=None, swap=None):
    """float64: (ys, dx, dxls, {(p, name): (dA, dB)}).  `drop_problem` leaves that problem's LoRA term out of dx, `swap`
    = (a, b) gives adapter a's rows adapter b's weights: the negative controls."""
    rn = lambda t: t.to(cdt).double()  # noqa: E731
    x64 = x.double()
    na = len(adapters[0])
    names = list(adapters[0])
    use = rows.long().clone()
    if swap is not None:
        use[rows.long() == swap[0]] = swap[1]
    base = sum(d.double() @ w for d, w in zip(dys, w64s))
    lora_dx = torch.zeros_like(base)
    ys, dxls, grads = [], [], {}
    for p, (ad, dy, w64) in enumerate(zip(adapters, dys, w64s)):
        xl = x64 if xls is None else xls[p].double()
        y = x64 @ w64.t()
        dxl = torch.zeros_like(x64)
        dy64 = dy.double()
        for i, name in enumerate(names):
            a, b, s = (t.detach().double() if torch.is_tensor(t) else t for t in ad[name])
            own = (rows.long() == i).nonzero().flatten()
            sel = (use == i).nonzero().flatten()
            if sel.numel():
                u = rn(s * (xl[sel] @ a.t()))
                y[sel] += u @ b.t()
                g = rn(s * (dy64[sel] @ b))
                if p != drop_problem:
                    lora_dx[sel] += g @ a
                dxl[sel] = g @ a
            # the gradient of adapter i comes from its own rows (the control swaps the weights those rows read)
            if own.numel():
                ai, bi, si = (t.detach().double() if torch.is_tensor(t) else t for t in ad[names[int(use[own[0]])]])
                u = rn(si * (xl[own] @ ai.t()))
                g = rn(si * (dy64[own] @ bi))
                grads[(p, name)] = (g.t() @ xl[own], dy64[own].t() @ u)
            else:
                grads[(p, name)] = (torch.zeros_like(a), torch.zeros_like(b))
        ys.append(y)
        dxls.append(dxl)
    dx = rn(rn(base) + lora_dx)
    return ys, dx, dxls, grads


def _run(x, bases, sets, rows, dys, x_loras=None):
    q = _q()
    x = x.detach().requires_grad_()
    xls = None if x_loras is None else [t.detach().requires_grad_() for t in x_loras]
    for s in sets:
        for t in s.lora_as + s.lora_bs:
            t.grad = None
    ys = q.lora_linear4bit_group_multi(x, bases, sets, rows, xls)
    torch.autograd.backward(ys, dys)
    return ys, x.grad, None if xls is None else [t.grad for t in xls]


# ---- forward bits --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cdt_name", ["bf16", "fp16"])
def test_forward_is_the_segmented_mixed_forward(c_oracle, cdt_name):
    """Above 16 rows the forward is `lora_linear4bit_group_mixed`'s tensor form bit for bit (U from the mixed projection
    below 768 rows x problems, from the shrink above); at 16 rows and below (where the mixed form runs the skinny decode
    kernels) it stays within the float64 bound of the segmented path."""
    q = _q()
    bases, adapters, sets, cdt, sdt = _setup("qkv", cdt_name, 16)
    w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
    for m in (17, 300, 1600):
        x = make_act(m, 4096, seed=m).to(cdt)
        rows = _rows(m, 16)
        ys = q.lora_linear4bit_group_multi(x, bases, sets, rows)
        with torch.no_grad():
            want = q.lora_linear4bit_group_mixed(x, bases, sets, rows)
        for y, w in zip(ys, want):
            assert torch.equal(y, w), m
    for m in (1, 16):
        x = make_act(m, 4096, seed=m).to(cdt)
        rows = _rows(m, 16)
        ys = q.lora_linear4bit_group_multi(x, bases, sets, rows)
        ref = _reference(x, None, [torch.zeros(m, 4096, dtype=cdt, device="cuda")] * 3, w64s, adapters, rows, cdt)[0]
        for y, r in zip(ys, ref):
            _check(y, r.to(cdt).double(), f"y m={m}", tol=4e-3 if cdt == BF16 else TOL)


# ---- gradients against float64 ---------------------------------------------------------------------------------------------

CASES = [(g, c) for g in ("qkv", "gate_up", "down") for c in ("bf16", "fp16")] + [("qkv", "bf16_over_fp16_state"),
                                                                                   ("ragged", "bf16")]


@pytest.mark.parametrize("dropout", [False, True], ids=["x", "x_loras"])
@pytest.mark.parametrize("group,cdt_name", CASES)
def test_gradients_match_float64(c_oracle, group, cdt_name, dropout):
    n, k, p = SHAPES[group]
    for na, m in ((1, 300), (4, 1600), (64, 700)):
        bases, adapters, sets, cdt, sdt = _setup(group, cdt_name, na, seed=na)
        w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
        x = make_act(m, k, seed=m + na).to(cdt)
        x_loras = [make_act(m, k, seed=m + 7 * i + 1).to(cdt) for i in range(p)] if dropout else None
        rows = _rows(m, na, seed=na)
        dys = [make_act(m, n, seed=3 * i + na).to(cdt) for i in range(p)]
        ys, dx, dxls = _run(x, bases, sets, rows, dys, x_loras)
        ref_y, ref_dx, ref_dxls, grads = _reference(x, x_loras, dys, w64s, adapters, rows, cdt)
        tag = f"{group} {cdt_name} na={na} m={m}"
        for y, r in zip(ys, ref_y):
            _check(y, r.to(cdt).double(), "y " + tag, tol=2.5e-3 if cdt == BF16 else TOL)
        if dropout:
            # x feeds the base only: dx is the base dX launch; each dropped input gets its own problem's LoRA term
            ref_base = sum(d.double() @ w for d, w in zip(dys, w64s)).to(cdt).double()
            _check(dx, ref_base, "dx " + tag)
            for i in range(p):
                _check(dxls[i], ref_dxls[i].to(cdt).double(), f"dxl{i} " + tag)
        else:
            _check(dx, ref_dx, "dx " + tag)
        for i, (s, ad) in enumerate(zip(sets, adapters)):
            for a_i, name in enumerate(s.names):
                da, db = grads[(i, name)]
                ga, gb = ad[name][0].grad, ad[name][1].grad
                assert ga.shape == ad[name][0].shape and gb.shape == ad[name][1].shape
                if not (rows == a_i).any():
                    assert not ga.any() and not gb.any(), f"absent adapter {name} " + tag
                    continue
                tol = TOL_WGRAD_BF16 if cdt == BF16 else TOL
                _check(ga, da.to(cdt).double(), f"dA p{i} {name} " + tag, tol=tol)
                _check(gb, db.to(cdt).double(), f"dB p{i} {name} " + tag, tol=tol)


def test_global_histogram_table(c_oracle):
    """More adapters than the segment table's shared-memory histogram holds (6015): rank-8 adapters at the ragged shape."""
    na, m = 6100, 900
    bases, adapters, sets, cdt, sdt = _setup("ragged", "bf16", na, seed=5, ranks=[8])
    n, k, p = SHAPES["ragged"]
    w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
    x = make_act(m, k, seed=1).to(cdt)
    rows = torch.tensor([-1 if t % 5 == 0 else (6007 * t) % na for t in range(m)], dtype=torch.int32, device="cuda")
    dys = [make_act(m, n, seed=2 + i).to(cdt) for i in range(p)]
    ys, dx, _ = _run(x, bases, sets, rows, dys)
    ref_y, ref_dx, _, grads = _reference(x, None, dys, w64s, adapters, rows, cdt)
    _check(dx, ref_dx, "dx")
    present = sorted(set(rows[rows >= 0].tolist()))
    for i, ad in enumerate(adapters):
        for a_i in present[::7] + [present[-1]]:
            name = f"ad{a_i}"
            da, db = grads[(i, name)]
            _check(ad[name][0].grad, da.to(cdt).double(), f"dA {name}", tol=TOL_WGRAD_BF16)
            _check(ad[name][1].grad, db.to(cdt).double(), f"dB {name}", tol=TOL_WGRAD_BF16)
    absent = next(a for a in range(na) if a not in set(present))
    assert not adapters[0][f"ad{absent}"][0].grad.any() and not adapters[0][f"ad{absent}"][1].grad.any()


# ---- negative controls ------------------------------------------------------------------------------------------------------

def test_negative_controls_exceed_the_bounds(c_oracle):
    bases, adapters, sets, cdt, sdt = _setup("qkv", "bf16", 4, seed=9, ranks=[16])
    w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
    m = 600
    x = make_act(m, 4096, seed=3).to(cdt)
    rows = _rows(m, 4)
    dys = [make_act(m, 4096, seed=10 + i).to(cdt) for i in range(3)]
    _, dx, _ = _run(x, bases, sets, rows, dys)
    grads_ok = {(i, nm): (ad[nm][0].grad.clone(), ad[nm][1].grad.clone()) for i, ad in enumerate(adapters) for nm in ad}
    _, ref_dx, _, _ = _reference(x, None, dys, w64s, adapters, rows, cdt, drop_problem=1)
    with pytest.raises(AssertionError):
        _check(dx, ref_dx, "dx without problem 1's LoRA term")
    _, ref_dx, _, grads = _reference(x, None, dys, w64s, adapters, rows, cdt, swap=(2, 3))
    with pytest.raises(AssertionError):
        _check(dx, ref_dx, "dx with adapter 3 on adapter 2's rows")
    with pytest.raises(AssertionError):
        _check(grads_ok[(0, "ad2")][0], grads[(0, "ad2")][0].to(cdt).double(), "dA with adapter 3 on adapter 2's rows",
               tol=TOL_WGRAD_BF16)


# ---- equivalence with training each adapter alone -------------------------------------------------------------------------

@pytest.mark.parametrize("group", ["qkv", "gate_up"])
def test_each_adapter_gets_the_gradient_of_its_rows_alone(group):
    q = _q()
    n, k, p = SHAPES[group]
    bases, adapters, sets, cdt, _ = _setup(group, "bf16", 4, seed=11, ranks=[16, 72, 16, 256])
    m = 1200
    x = make_act(m, k, seed=5).to(cdt)
    rows = _rows(m, 4)
    dys = [make_act(m, n, seed=20 + i).to(cdt) for i in range(p)]
    _run(x, bases, sets, rows, dys)
    for i_a, name in enumerate(sets[0].names):
        sel = (rows == i_a).nonzero().flatten()
        a_s = [ad[name][0].detach().clone().requires_grad_() for ad in adapters]
        b_s = [ad[name][1].detach().clone().requires_grad_() for ad in adapters]
        ys = q.lora_linear4bit_group(x[sel], bases, a_s, b_s, adapters[0][name][2])
        torch.autograd.backward(ys, [d[sel] for d in dys])
        for ip, ad in enumerate(adapters):
            _check(ad[name][0].grad, a_s[ip].grad.double(), f"dA {name} p{ip}", tol=TOL_WGRAD_BF16)
            _check(ad[name][1].grad, b_s[ip].grad.double(), f"dB {name} p{ip}", tol=TOL_WGRAD_BF16)


# ---- edge rows, determinism, no sync, reads inside operands ----------------------------------------------------------------

def test_base_and_out_of_range_rows_take_the_base_dx_bits():
    q = _q()
    F = q.functional
    bases, adapters, sets, cdt, _ = _setup("qkv", "bf16", 8, seed=13)
    m = 700
    idx = [(t % 11) - 2 for t in range(m)]                     # -2, -1, 0..8: 8 is out of range for 8 adapters
    idx[3::13] = [1 << 30] * len(idx[3::13])
    rows = torch.tensor(idx, dtype=torch.int32, device="cuda")
    x = make_act(m, 4096, seed=7).to(cdt)
    dys = [make_act(m, 4096, seed=30 + i).to(cdt) for i in range(3)]
    _, dx, _ = _run(x, bases, sets, rows, dys)
    base_dx = F.nf4_linear_group(True, dys, [b.weight.t() for b in bases], [b.weight.quant_state for b in bases], out_dtype=cdt)
    none = (rows < 0) | (rows >= 8)
    assert torch.equal(dx[none], base_dx[none])
    assert not torch.equal(dx[~none], base_dx[~none])


def test_two_calls_give_the_same_bits_and_no_host_sync():
    bases, adapters, sets, cdt, _ = _setup("gate_up", "bf16", 4, seed=17)
    m = 1000
    x = make_act(m, 4096, seed=8).to(cdt)
    rows = _rows(m, 4)
    dys = [make_act(m, 11008, seed=40 + i).to(cdt) for i in range(2)]
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            ys, dx, _ = _run(x, bases, sets, rows, dys)
            runs.append((ys, dx, [t.grad.clone() for s in sets for t in s.lora_as + s.lora_bs]))
        for a, b in zip(runs[0][0] + (runs[0][1],) + tuple(runs[0][2]), runs[1][0] + (runs[1][1],) + tuple(runs[1][2])):
            assert torch.equal(a, b)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            _run(x, bases, sets, rows, dys)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        torch.use_deterministic_algorithms(False)


def test_reads_stay_inside_operands():
    """Adapters inside NaN-filled buffers, row indices whose neighbours in memory point far outside the table: every output
    is finite and equal to the call on clean copies."""
    q = _q()
    n, k = 1000, 1088
    cdt = BF16
    bases = [_base(n, k, cdt, cdt, seed=50 + i) for i in range(2)]
    clean = [_adapters(n, k, 5, cdt, seed=700 + i) for i in range(2)]
    padded = []
    for ad in clean:
        out = {}
        for name, (a, b, s) in ad.items():
            ba = torch.full((a.numel() + 2 * k,), float("nan"), dtype=cdt, device="cuda")
            bb = torch.full((b.numel() + 64,), float("nan"), dtype=cdt, device="cuda")
            ba[k:k + a.numel()] = a.detach().flatten()
            bb[32:32 + b.numel()] = b.detach().flatten()
            out[name] = (ba[k:k + a.numel()].view_as(a).requires_grad_(), bb[32:32 + b.numel()].view_as(b).requires_grad_(), s)
        padded.append(out)
    m = 333
    buf = torch.full((m + 64,), 1 << 30, dtype=torch.int32, device="cuda")
    buf[32:32 + m] = _rows(m, 5)
    rows = buf[32:32 + m]
    x = make_act(m, k, seed=9).to(cdt)
    dys = [make_act(m, n, seed=60 + i).to(cdt) for i in range(2)]
    got = _run(x, bases, [q.LoraAdapterSet(a) for a in padded], rows, dys)
    want = _run(x, bases, [q.LoraAdapterSet(a) for a in clean], rows.clone(), dys)
    for g, w in zip(list(got[0]) + [got[1]], list(want[0]) + [want[1]]):
        assert torch.isfinite(g).all() and torch.equal(g, w)
    for pa, ca in zip(padded, clean):
        for name in pa:
            for j in (0, 1):
                assert torch.isfinite(pa[name][j].grad).all() and torch.equal(pa[name][j].grad, ca[name][j].grad)


# ---- a toy two-block model: CUDA graph, torch.compile, one training step ------------------------------------------------

class _Toy(torch.nn.Module):
    """Two Llama-like blocks (q/k/v grouped, o, gate/up grouped, down, SiLU), every linear an NF4 base with K adapters."""

    def __init__(self, d, f, na, cdt, seed):
        super().__init__()
        q = _q()
        self.blocks = []
        s = seed
        for _ in range(2):
            blk = {}
            for name, (n, k, cnt) in {"qkv": (d, d, 3), "o": (d, d, 1), "gu": (f, d, 2), "down": (d, f, 1)}.items():
                bases = [_base(n, k, cdt, cdt, seed=s + i) for i in range(cnt)]
                ads = [_adapters(n, k, na, cdt, seed=100 * s + 10 * i, ranks=[16, 8]) for i in range(cnt)]
                blk[name] = (bases, ads, [q.LoraAdapterSet(a) for a in ads])
                s += 7
            self.blocks.append(blk)

    def params(self):
        return [t for blk in self.blocks for (_, ads, _) in blk.values() for ad in ads for (a, b, _) in ad.values() for t in (a, b)]

    def forward(self, x, rows):
        q = _q()
        multi = q.lora_linear4bit_group_multi
        for blk in self.blocks:
            qq, kk, vv = multi(x, blk["qkv"][0], blk["qkv"][2], rows)
            h = x + multi(qq * kk + vv, blk["o"][0], blk["o"][2], rows)[0]
            g, u = multi(h, blk["gu"][0], blk["gu"][2], rows)
            x = h + multi(torch.nn.functional.silu(g) * u, blk["down"][0], blk["down"][2], rows)[0]
        return x


def _step(model, x, rows, dy):
    for t in model.params():
        t.grad = None
    y = model(x, rows)
    y.backward(dy)
    return y


def test_cuda_graph_replay_follows_the_index_buffer():
    model = _Toy(512, 1024, 4, BF16, seed=3)
    m = 256
    x = make_act(m, 512, seed=1).requires_grad_()
    dy = make_act(m, 512, seed=2)
    rows_buf = _rows(m, 4)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _step(model, x, rows_buf, dy)
    torch.cuda.current_stream().wait_stream(side)
    for t in model.params():                                # graph-owned gradient buffers
        t.grad = None
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = model(x, rows_buf)
        grads = torch.autograd.grad(y, [x] + model.params(), dy)
    for seed in (5, 6):
        new = _rows(m, 4, seed=seed)
        new[::5] = -1
        rows_buf.copy_(new)
        graph.replay()
        torch.cuda.synchronize()
        y_eager = model(x, new)
        g_eager = torch.autograd.grad(y_eager, [x] + model.params(), dy)
        assert torch.equal(y, y_eager)
        for a, b in zip(grads, g_eager):
            assert torch.equal(a, b)


def test_compiled_step_is_one_graph():
    """fullgraph=True: the toy model's forward traces without a graph break and its backward is traced with it; the aot_eager
    backend runs the same ops, so the step gives eager's bits."""
    model = _Toy(512, 1024, 4, BF16, seed=4)
    m = 320
    x = make_act(m, 512, seed=1)
    dy = make_act(m, 512, seed=2)
    rows = _rows(m, 4)
    runs = []
    torch._dynamo.reset()
    for fwd in (torch.compile(model.forward, fullgraph=True, backend="aot_eager"), model.forward):
        xr = x.detach().requires_grad_()
        for t in model.params():
            t.grad = None
        y = fwd(xr, rows)
        y.backward(dy)
        runs.append([y, xr.grad] + [t.grad for t in model.params()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_training_step_per_job_matches_training_alone():
    """K = 4 jobs in one batch, each loss the mean over its own tokens, one library AdamW per adapter: after one step each
    adapter's weights are within the float64 bound of the same step run on that adapter's rows alone (the toy model mixes
    no rows, so each adapter's gradient comes from its own rows only)."""
    q = _q()
    na, seq = 4, 96
    model = _Toy(512, 1024, na, BF16, seed=6)
    m = na * seq
    x = make_act(m, 512, seed=3)
    target = make_act(m, 512, seed=4)
    rows = torch.arange(na, device="cuda", dtype=torch.int32).repeat_interleave(seq)
    params = model.params()
    by_adapter = {a: [] for a in range(na)}
    for blk in model.blocks:
        for (_, ads, _) in blk.values():
            for ad in ads:
                for i, (a_, b_, _) in enumerate(ad.values()):
                    by_adapter[i] += [a_, b_]
    before = [t.detach().clone() for t in params]

    def step(sel_rows, jobs):
        for t in params:
            t.grad = None
        y = model(x[sel_rows], rows[sel_rows])
        loss = sum(((y[rows[sel_rows] == a].float() - target[sel_rows][rows[sel_rows] == a].float()) ** 2).mean() for a in jobs)
        loss.backward()
        for a in jobs:
            q.optim.AdamW(by_adapter[a], lr=1e-3).step()

    step(torch.arange(m, device="cuda"), range(na))
    together = {id(t): t.detach().clone() for t in params}
    for a in range(na):
        with torch.no_grad():
            for t, b0 in zip(params, before):
                t.copy_(b0)
        step((rows == a).nonzero().flatten(), [a])
        for t in by_adapter[a]:
            # AdamW's first step moves each element by about lr . sign(g), so an element whose g is within rounding noise of
            # zero can step the other way in one of the runs (2 lr apart, 3 bf16 ulp of max|weight| measured): the bound is
            # on the Frobenius norm only (4.3e-4 measured on an H100)
            _check(together[id(t)], t.detach().double(), f"adapter {a} after one step", ulps=float("inf"))
