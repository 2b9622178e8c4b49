"""The segmented LoRA kernels (qlora_b200/csrc/lora_segmented.cu) at the layouts where they can go wrong: bucket sizes at and
around the 64-row tile and the weight gradient's 64-row chunks, the segment table's 1024-bucket scan chunks and its
shared/global histogram switch, grouped problems whose ranks differ, and both sides of the host's thresholds.

* The segment table, bit for bit: the workspace `lora_segmented_fwd` returns, decoded with a restatement of seg::layout,
  against a host restatement (stable argsort of the buckets, exclusive prefix sum, tiles of at most 64 rows, zero padding up
  to ceil(M / 64) + n tiles).  No tolerance.
* The mixed forward (`lora_linear4bit_group_mixed`) against float64 (`_ref` of tests/test_gpu_mixed_adapters.py): adapter a
  has rank 8, 256 and 72 in the three problems of a q/k/v group (R = 256: U tiles of columns [128, 256) of the rank-8 and
  rank-72 problems take the shrink's zero-fill branch, and the expand's contraction stops at each problem's own rank), at
  rows x problems = SEGMENTED_SHRINK_MIN_WORK - 1 and SEGMENTED_SHRINK_MIN_WORK (U from `lora_project_mixed`, then from the
  segmented shrink).  The names form at ranks adding up to 256 in every set, and to 264 in one.
* Training (`lora_linear4bit_group_multi`) against float64 (`_reference` of tests/test_gpu_multi_adapter_train.py), with and
  without dropped inputs: buckets of 1, 63, 64, 65, 128 and 129 rows at ranks 8, 72, 136 and 256; every row on one adapter;
  no adapter row at all, where dA and dB are exactly zero and y and dx are the base launches' bits.

Bounds.  As in tests/test_gpu_multi_adapter_train.py, the reference rounds where the definition rounds, and a result then
differs from it only where the kernel's fp32 sum and the float64 sum straddle a rounding boundary: one ulp of that element,
on about 2^-24 sqrt(N) / 2^-8 (well under 1 %) of the elements.  One ulp is at most 2^-8 (bf16) or 2^-11 (fp16) of an
element, so 1e-3 Frobenius-relative allows a flip on 6.5 % of the elements.  Every element must also be within 1.01 ulp of
max|ref|, in the compute dtype's own ulp (2^-7 of the top binade for bf16, 2^-10 for fp16).
  - y of the segmented forward (tensor form and training): the path rounds the base output, then the sum with the LoRA
    term, so the reference is `_twice_rounded`: rn(rn(x W^T) + LoRA term) on `_ref` / `_reference`; bar 1e-3.  Against the
    once-rounded reference the second rounding moves about a quarter of the elements of every row with an adapter by one
    ulp: SEG_TOL_BF16 (2.5e-3, tests/test_gpu_mixed_segmented.py) was measured with a third of the rows on the base, and
    with every row on an adapter the bf16 error grows by sqrt(3/2), to 2.85e-3 measured (each element still within 1.00
    ulp).  Against the twice-rounded reference: 2.9e-4 (tensor form) and 3.1e-4 (training) measured under bf16, 1.1e-4
    and 4.7e-5 under fp16.
  - y of the names form (one rounding) against `_ref`: 1e-3; 1.3e-4 measured (fp16 5.0e-5).
  - dx and dxl: 1e-3, as tests/test_gpu_multi_adapter_train.py; 3.9e-4 and 4.5e-4 measured (fp16 7.5e-5 and 8.3e-5).
  - dA and dB: with one to a few rows per adapter, one flipped element of G (or U) is a large share of that adapter's dA
    (dB) rows, so a Frobenius bound per adapter is noise.  Instead: each element within 1.01 ulp of max|ref| of that
    adapter's block (per problem), and a Frobenius-relative bound over all adapters and problems together, TOL_WGRAD_BF16 =
    2.5e-3 (bf16) or 1e-3 (fp16).  For a one-row adapter, dA_a = g^T x_t: a G element g_i off by its own ulp moves element
    (i, j) by ulp(g_i) |x_j|, under two ulp of that element, but only on the rare flipped g_i.  Measured: every element
    within 1.00 ulp of its block's max; over all adapters 4.6e-4 (bf16) and 8.3e-5 (fp16); the worst single block
    9.4e-4 (bf16), the noise a per-adapter Frobenius bound would have to absorb.
Measured on an H100 80GB HBM3 at 700 W.

Negative controls must miss their bar by CONTROL_MARGIN (10x).  A reference that moves the first row of ad3's 65-row
bucket into the previous bucket: y 3.0e-2 (30x) and 86 ulp; dA and dB of ad2 and ad3 1.1e-1 to 1.3e-1 (43x to 52x) and 33
to 57 ulp.  A forward reference that gives every problem problem 0's ranks: problems 1 and 2 at 3.2e-1 and 3.8e-1 (over
300x) and 159 and 181 ulp.
"""
import numpy as np
import pytest
import torch

from gpu_helpers import make_act, make_weight, rel_err
from test_gpu_mixed_adapters import _base as _mixed_base
from test_gpu_mixed_adapters import _ref
from test_gpu_mixed_adapters import _w64 as _mixed_w64
from test_gpu_multi_adapter_train import SHAPES, TOL, TOL_WGRAD_BF16, _reference, _run, _setup, _w64

pytestmark = pytest.mark.gpu

BF16, H16 = torch.bfloat16, torch.float16
NO_ADAPTER = (-1, None, 1 << 30)          # None: n, the first index past the table
EDGE_BUCKETS = (63, 64, 65, 128, 129)
CONTROL_MARGIN = 10.0                     # a negative control misses its bar by at least this factor


def _q():
    import qlora_b200 as q

    return q


# ---- errors against a float64 reference ---------------------------------------------------------------------------------

def _ulps(got: np.ndarray, want: np.ndarray, cdt) -> float:
    """max |got - want| in ulps of the compute dtype at the top binade of max|want|."""
    scale = max(float(np.abs(want).max()), 1e-30)
    ulp = 2.0 ** (np.floor(np.log2(scale)) - (7 if cdt == BF16 else 10))
    return float(np.abs(got.astype(np.float64) - want.astype(np.float64)).max() / ulp)


class _Bars:
    """Collects every comparison of a test and fails at the end with all that missed, so one run reports each case's error."""

    def __init__(self, record):
        self.record, self.fails, self.worst = record, [], {}

    def check(self, got, ref, cdt, what, tol, ulps=1.01, kind=None):
        """got against ref rounded to cdt: rel_F <= tol and each element within `ulps`; returns (rel_F, ulps)."""
        g = got.detach().float().cpu().numpy()
        w = ref.to(cdt).float().cpu().numpy()
        e, u = rel_err(g, w), _ulps(g, w, cdt)
        self._note(kind or what.split()[0], e, u)
        if not (e <= tol and u <= ulps):
            self.fails.append(f"{what}: rel_F={e:.3e} (bar {tol:.1e}), max err {u:.2f} ulp (bar {ulps})")
        return e, u

    def _note(self, kind, e, u):
        we, wu = self.worst.get(kind, (0.0, 0.0))
        self.worst[kind] = (max(we, e), max(wu, u))

    def done(self):
        for kind, (e, u) in sorted(self.worst.items()):
            self.record(f"worst {kind}", f"rel_F={e:.3e} ulp={u:.3f}")
        assert not self.fails, "\n".join(self.fails)


@pytest.fixture
def bars(record_property):
    return _Bars(record_property)


def _twice_rounded(ref, base64, cdt):
    """The segmented forward's two roundings restated on a float64 reference `ref` of x W^T + LoRA term: rn(rn(x W^T) + LoRA
    term), the term being ref - x W^T (exactly zero on rows without an adapter, which keep rn(x W^T))."""
    return (base64.to(cdt).double() + (ref - base64)).to(cdt).double()


def _errs(got, ref, cdt):
    g = got.detach().float().cpu().numpy()
    w = ref.to(cdt).float().cpu().numpy()
    return rel_err(g, w), _ulps(g, w, cdt)


# ---- row layouts ---------------------------------------------------------------------------------------------------------

def _no_adapter(t, n):
    v = NO_ADAPTER[t % 3]
    return n if v is None else v


def _bucket_rows(sizes, ids, m, n, seed):
    """int32 [m] on the host: sizes[i] rows on adapter ids[i] (truncated to m), the rest cycling through indices that mean no
    adapter (-1, n, 2^30), in an order shuffled by `seed` so the sort has to be stable to keep row order."""
    idx = [a for s, a in zip(sizes, ids) for _ in range(s)][:m]
    idx += [_no_adapter(t, n) for t in range(m - len(idx))]
    return np.asarray(idx, np.int64)[np.random.default_rng(seed).permutation(m)].astype(np.int32)


def _table_layout(kind, m, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "one":
        return np.full(m, n - 1, np.int32)
    if kind == "none":
        return np.asarray([_no_adapter(t, n) for t in range(m)], np.int32)
    if kind == "one_per_adapter":                      # distinct adapters while m <= n
        return (rng.permutation(max(m, n))[:m] % n).astype(np.int32)
    ids = rng.permutation(n)[:len(EDGE_BUCKETS)] if n >= len(EDGE_BUCKETS) else [i % n for i in range(len(EDGE_BUCKETS))]
    return _bucket_rows(EDGE_BUCKETS, ids, m, n, seed)


# ---- 1. the segment table, bit for bit ------------------------------------------------------------------------------------

def _table_ref(idx, n):
    """The segment table restated: (perm [M], off [n + 2], tiles [ceil(M / 64) + n, 4]) as int32."""
    m = len(idx)
    b = np.where((idx >= 0) & (idx < n), idx, n).astype(np.int64)
    perm = np.argsort(b, kind="stable")
    off = np.zeros(n + 2, np.int64)
    off[1:] = np.cumsum(np.bincount(b, minlength=n + 1))
    tiles = np.zeros(((m + 63) // 64 + n, 4), np.int64)
    j = 0
    for a in np.flatnonzero(off[1:n + 1] > off[:n]):
        for first in range(off[a], off[a + 1], 64):
            tiles[j] = (a, first, min(64, off[a + 1] - first), 0)
            j += 1
    return perm.astype(np.int32), off.astype(np.int32), tiles.astype(np.int32)


def _table_decode(ws: np.ndarray, m, n):
    """seg::layout(M, n): perm at 0, offsets at align16(4 M), tiles after align16(4 (n + 2)) more bytes."""
    a16 = lambda b: (b + 15) // 16 * 16  # noqa: E731
    off0 = a16(4 * m)
    t0 = off0 + a16(4 * (n + 2))
    n_tiles = (m + 63) // 64 + n
    return (ws[:4 * m].view(np.int32), ws[off0:off0 + 4 * (n + 2)].view(np.int32),
            ws[t0:t0 + 16 * n_tiles].view(np.int32).reshape(n_tiles, 4))


TABLE_M = (1, 31, 32, 33, 64, 65, 1000)
TABLE_N = (1, 1023, 1024, 1025, 6015, 6016)


@pytest.mark.parametrize("n", TABLE_N)
def test_segment_table_is_the_stable_sort(n):
    """1023 and 1024 adapters: one scan chunk, and a second that holds only the "no adapter" bucket; 1025: two adapters' worth
    in the second.  6015: the largest table whose histogram is in shared memory; 6016: the global-memory histogram.  M of 31,
    32, 33 and 65 leave the scatter warp's last 32 rows partly empty.  The workspace comes from `lora_segmented_fwd`; a direct
    `qb200_lora_segment_table` into a workspace of 0xA5 bytes must write the same perm, offsets and tiles, so the zero tiles
    are written by the kernel, not left over by the allocator."""
    q = _q()
    from qlora_b200 import _lib, _ops

    lib = _lib.load()
    k = 64
    g = torch.Generator().manual_seed(n)
    a_all = ((torch.rand(n * 8, k, generator=g) * 2 - 1) * 0.1).to(BF16).cuda()
    b_all = ((torch.rand(n, k, 8, generator=g) * 2 - 1) * 0.1).to(BF16).cuda()
    aset = q.LoraAdapterSet({f"ad{i}": (a_all[8 * i:8 * i + 8], b_all[i], 1.0) for i in range(n)})
    checked = 0
    for m in TABLE_M:
        nbytes = lib.qb200_lora_segment_workspace_size(m, n)
        assert nbytes == _ops.segment_workspace_bytes(m, n) > 0
        x = make_act(m, k, seed=m)
        for kind in ("one", "none", "edge_buckets", "one_per_adapter"):
            idx = _table_layout(kind, m, n, seed=1000 * m + n)
            rows = torch.from_numpy(idx).cuda()
            out = torch.zeros(m, k, dtype=BF16, device="cuda")
            with torch.no_grad():
                _, ws = _ops.lora_segmented_fwd([x], [aset.table], rows, n, 8, [out])
            poisoned = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device="cuda")
            _lib.check(lib.qb200_lora_segment_table(_lib.ptr(rows), m, n, _lib.ptr(poisoned), nbytes, _lib.stream_ptr(rows.device)),
                       "lora_segment_table")
            want = _table_ref(idx, n)
            for src in (ws, poisoned):
                got = _table_decode(src.cpu().numpy(), m, n)
                for part, a, b in zip(("perm", "off", "tiles"), got, want):
                    assert np.array_equal(a, b), f"{part}: n={n} m={m} {kind}"
            checked += 1
    assert checked == len(TABLE_M) * 4


# ---- 2. the mixed forward with unequal ranks across problems --------------------------------------------------------------

FWD_RANKS = (8, 256, 72)                  # adapter a has rank FWD_RANKS[(a + p) % 3] in problem p


def _adapter_sets(n, k, ranks, cdt, seed):
    """ranks[p][a]: one {name: (A, B, scaling)} per problem and its LoraAdapterSet; the same names in every problem."""
    q = _q()
    adapters = []
    for p, rp in enumerate(ranks):
        ad = {}
        for a, r in enumerate(rp):
            s = seed + 100 * p + 2 * a
            ad[f"ad{a}"] = (make_weight(r, k, seed=s, dtype=cdt, scale=k ** -0.5), make_weight(n, r, seed=s + 1, dtype=cdt, scale=0.05),
                            0.5 + 0.25 * ((a + p) % 3))
        adapters.append(ad)
    return adapters, [q.LoraAdapterSet(ad) for ad in adapters]


def _names(idx, na):
    return [f"ad{a}" if 0 <= a < na else "__base__" for a in idx.tolist()]


def _truncated(adapters, ranks):
    """The adapters cut to ranks[a] (the control that reads problem 0's ranks for every problem)."""
    return {nm: (a[:ranks[i]], b[:, :ranks[i]], s) for i, (nm, (a, b, s)) in enumerate(adapters.items())}


FWD_SHAPES = [(1000, 1088), (4096, 4096)]


@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,k", FWD_SHAPES, ids=[f"{n}x{k}" for n, k in FWD_SHAPES])
def test_tensor_form_unequal_ranks_matches_float64(c_oracle, bars, n, k, cdt):
    """q/k/v with 6 adapters of ranks (8, 256, 72) rotated over the problems; buckets of 63..129 rows, one-row buckets, every
    row on one adapter, on both sides of SEGMENTED_SHRINK_MIN_WORK for three problems and for one."""
    q = _q()
    from qlora_b200 import _ops

    na, p = 6, 3
    ranks = [[FWD_RANKS[(a + i) % 3] for a in range(na)] for i in range(p)]
    bases = [_mixed_base(n, k, cdt, seed=n + 13 * i) for i in range(p)]
    w64s = [_mixed_w64(b, c_oracle, cdt) for b in bases]
    adapters, sets = _adapter_sets(n, k, ranks, cdt, seed=n + k)
    work = _ops.SEGMENTED_SHRINK_MIN_WORK
    cases = []
    for nprob in (3, 1):
        lo, hi = (work - 1) // nprob, -(-work // nprob)          # rows x problems just below and at the threshold
        for m in (lo, hi):
            cases.append((nprob, m, _bucket_rows((63, 64, 65, 1, 1), range(5), m, na, seed=m)))
    cases.append((3, 1000, _bucket_rows(EDGE_BUCKETS + (1,), range(6), 1000, na, seed=7)))
    for m in (200, 300):                                          # below and above for three problems: every row on adapter 1
        cases.append((3, m, np.full(m, 1, np.int32)))
    for nprob, m, idx in cases:
        x = make_act(m, k, seed=m + nprob).to(cdt)
        names = _names(idx, na)
        with torch.no_grad():
            ys = q.lora_linear4bit_group_mixed(x, bases[:nprob], sets[:nprob], torch.from_numpy(idx).cuda())
        for i, y in enumerate(ys):
            tag = f"y p{i}/{nprob} m={m} {'shrink' if m * nprob >= work else 'project'}"
            base64 = x.double() @ w64s[i].t()
            bars.check(y, _twice_rounded(_ref(x, w64s[i], adapters[i], names, cdt), base64, cdt), cdt, tag, TOL, kind="y")
    bars.done()


@pytest.mark.parametrize("cdt", [BF16, H16], ids=["bf16", "fp16"])
def test_names_form_unequal_ranks_on_both_sides_of_the_rank_limit(c_oracle, bars, cdt):
    """Three problems whose three adapters have different ranks per problem: sums of 256 in every set (concat, one grouped
    launch), sums of 24, 256 and 88 (concat, one launch per problem: U widths differ), and a sum of 264 in one set (grouped:
    ad0 and ad1, then ad2).  One rounding, so the bar of the one-rounding paths (1e-3)."""
    q = _q()
    from qlora_b200.mixed import _rank_groups, prefill_branch

    n, k, m = 1000, 1088, 300
    bases = [_mixed_base(n, k, cdt, seed=40 + i) for i in range(3)]
    w64s = [_mixed_w64(b, c_oracle, cdt) for b in bases]
    variants = {"concat_256": ([128, 64, 64], [64, 128, 64], [64, 64, 128]),
                "concat_unequal_widths": ([8, 8, 8], [240, 8, 8], [72, 8, 8]),
                "grouped_264": ([128, 64, 64], [64, 128, 64], [64, 64, 136])}
    idx = _bucket_rows((63, 65, 129), range(3), m, 3, seed=3)
    names = _names(idx, 3)
    for v, ranks in variants.items():
        adapters, sets = _adapter_sets(n, k, ranks, cdt, seed=500)
        want = "grouped" if v == "grouped_264" else "concat"
        assert prefill_branch(sets, names) == want
        if want == "grouped":
            assert _rank_groups(sets, [0, 1, 2]) == [[0, 1], [2]]
        x = make_act(m, k, seed=9).to(cdt)
        with torch.no_grad():
            ys = q.lora_linear4bit_group_mixed(x, bases, sets, names)
        for i, y in enumerate(ys):
            bars.check(y, _ref(x, w64s[i], adapters[i], names, cdt), cdt, f"y {v} p{i}", TOL, kind="y")
    bars.done()


def test_control_problem0_ranks_misses_the_bar(c_oracle, record_property):
    """The forward reference with every problem cut to problem 0's ranks misses the bar of problems 1 and 2."""
    q = _q()
    n, k, na, m, cdt = 1000, 1088, 6, 1000, BF16
    ranks = [[FWD_RANKS[(a + i) % 3] for a in range(na)] for i in range(3)]
    bases = [_mixed_base(n, k, cdt, seed=n + 13 * i) for i in range(3)]
    adapters, sets = _adapter_sets(n, k, ranks, cdt, seed=n + k)
    idx = _bucket_rows(EDGE_BUCKETS + (1,), range(6), m, na, seed=7)
    names = _names(idx, na)
    x = make_act(m, k, seed=m + 3).to(cdt)
    with torch.no_grad():
        ys = q.lora_linear4bit_group_mixed(x, bases, sets, torch.from_numpy(idx).cuda())
    for i in (1, 2):
        w64 = _mixed_w64(bases[i], c_oracle, cdt)
        cut = _truncated(adapters[i], [min(a, b) for a, b in zip(ranks[0], ranks[i])])
        e, u = _errs(ys[i], _twice_rounded(_ref(x, w64, cut, names, cdt), x.double() @ w64.t(), cdt), cdt)
        record_property(f"problem {i}", f"rel_F={e:.3e} ulp={u:.2f}")
        assert max(e / TOL, u / 1.01) >= CONTROL_MARGIN, (i, e, u)


# ---- 3. training: buckets at the weight gradient's chunk edges --------------------------------------------------------------

TRAIN_RANKS = [8, 72, 136, 256]
# rows per adapter (adapter a has rank TRAIN_RANKS[a % 4]): ad3 (rank 256) holds 65 rows after ad2's 64, ad8 holds none
TRAIN_BUCKETS = (1, 63, 64, 65, 128, 129, 129, 1, 0)
TRAIN_CASES = [("ragged", "bf16"), ("ragged", "fp16"), ("qkv", "bf16")]


def _train_layouts(na):
    m = 900
    return {"edge_buckets": _bucket_rows(TRAIN_BUCKETS, range(na), m, na, seed=11),
            "one_adapter": np.full(300, 3, np.int32),
            "no_adapter": np.asarray([_no_adapter(t, na) for t in range(300)], np.int32)}


def _wgrad_check(bars, adapters, grads, idx, cdt, tag):
    """dA and dB: each adapter block's elements within 1.01 ulp of its own max|ref|, and rel_F over all blocks together."""
    tol = TOL_WGRAD_BF16 if cdt == BF16 else TOL
    num = {"dA": 0.0, "dB": 0.0}
    den = {"dA": 0.0, "dB": 0.0}
    for p, ad in enumerate(adapters):
        for a, name in enumerate(ad):
            for j, kind in enumerate(("dA", "dB")):
                got = ad[name][j].grad
                want = grads[(p, name)][j]
                assert got.shape == want.shape
                if not (idx == a).any():
                    if got.count_nonzero():
                        bars.fails.append(f"{kind} of absent {name} p{p} {tag}: not zero")
                    continue
                g, w = got.double(), want.to(cdt).double()
                num[kind] += float(((g - w) ** 2).sum())
                den[kind] += float((w ** 2).sum())
                bars.check(got, want, cdt, f"{kind} p{p} {name} ({int((idx == a).sum())} rows) {tag}", float("inf"),
                           kind=f"{kind} block")
    for kind in ("dA", "dB"):
        e = (num[kind] / max(den[kind], 1e-300)) ** 0.5
        bars._note(f"{kind} all", e, 0.0)
        if e > tol:
            bars.fails.append(f"{kind} over all adapters {tag}: rel_F={e:.3e} (bar {tol:.1e})")


@pytest.mark.parametrize("dropout", [False, True], ids=["x", "x_loras"])
@pytest.mark.parametrize("group,cdt_name", TRAIN_CASES)
def test_training_at_bucket_edges_matches_float64(c_oracle, bars, group, cdt_name, dropout):
    q = _q()
    F = q.functional
    n, k, p = SHAPES[group]
    na = len(TRAIN_BUCKETS)
    bases, adapters, sets, cdt, sdt = _setup(group, cdt_name, na, seed=3, ranks=TRAIN_RANKS)
    w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
    for lay, idx in _train_layouts(na).items():
        m = len(idx)
        rows = torch.from_numpy(idx).cuda()
        x = make_act(m, k, seed=m + 1).to(cdt)
        x_loras = [make_act(m, k, seed=m + 7 * i + 2).to(cdt) for i in range(p)] if dropout else None
        dys = [make_act(m, n, seed=5 * i + m).to(cdt) for i in range(p)]
        ys, dx, dxls = _run(x, bases, sets, rows, dys, x_loras)
        tag = f"{lay} m={m}"
        if lay == "no_adapter":
            base_y = F.nf4_linear_group(False, [x] * p, [b.weight.t() for b in bases], [b.weight.quant_state for b in bases])
            base_dx = F.nf4_linear_group(True, dys, [b.weight.t() for b in bases], [b.weight.quant_state for b in bases],
                                         out_dtype=cdt)
            assert all(torch.equal(y, b) for y, b in zip(ys, base_y)), "y with no adapter row"
            assert torch.equal(dx, base_dx), "dx with no adapter row"
            if dropout:
                assert not any(t.count_nonzero() for t in dxls), "dxl with no adapter row"
            for s in sets:
                assert not any(t.grad.count_nonzero() for t in s.lora_as + s.lora_bs), "dA, dB with no adapter row"
            continue
        ref_y, ref_dx, ref_dxls, grads = _reference(x, x_loras, dys, w64s, adapters, rows, cdt)
        for i, (y, r) in enumerate(zip(ys, ref_y)):
            bars.check(y, _twice_rounded(r, x.double() @ w64s[i].t(), cdt), cdt, f"y p{i} {tag}", TOL)
        if dropout:
            bars.check(dx, sum(d.double() @ w for d, w in zip(dys, w64s)), cdt, f"dx {tag}", TOL)
            for i in range(p):
                bars.check(dxls[i], ref_dxls[i], cdt, f"dxl p{i} {tag}", TOL)
        else:
            bars.check(dx, ref_dx, cdt, f"dx {tag}", TOL)
        _wgrad_check(bars, adapters, grads, idx, cdt, tag)
    bars.done()


def test_control_moved_row_misses_the_bar(c_oracle, record_property):
    """The reference with the first sorted row of ad3's 65-row bucket moved into the previous bucket (ad2's 64 rows): y of
    that row, and dA / dB of ad2 and ad3, miss their bars."""
    n, k, p = SHAPES["ragged"]
    na = len(TRAIN_BUCKETS)
    bases, adapters, sets, cdt, sdt = _setup("ragged", "bf16", na, seed=3, ranks=TRAIN_RANKS)
    w64s = [_w64(b, c_oracle, cdt, sdt) for b in bases]
    idx = _train_layouts(na)["edge_buckets"]
    m = len(idx)
    rows = torch.from_numpy(idx).cuda()
    x = make_act(m, k, seed=m + 1).to(cdt)
    dys = [make_act(m, n, seed=5 * i + m).to(cdt) for i in range(p)]
    ys, _, _ = _run(x, bases, sets, rows, dys)
    moved = rows.clone()
    first = int((rows == 3).nonzero().flatten()[0])
    moved[first] = 2
    ref_y, _, _, grads = _reference(x, None, dys, w64s, adapters, moved, cdt)
    e, u = _errs(ys[0], _twice_rounded(ref_y[0], x.double() @ w64s[0].t(), cdt), cdt)
    record_property("y", f"rel_F={e:.3e} ulp={u:.2f}")
    assert max(e / TOL, u / 1.01) >= CONTROL_MARGIN, ("y", e, u)
    for name in ("ad2", "ad3"):
        for j, kind in enumerate(("dA", "dB")):
            e, u = _errs(adapters[0][name][j].grad, grads[(0, name)][j], cdt)
            record_property(f"{kind} {name}", f"rel_F={e:.3e} ulp={u:.2f}")
            assert max(e / TOL_WGRAD_BF16, u / 1.01) >= CONTROL_MARGIN, (kind, name, e, u)


def test_multi_refuses_unequal_ranks_across_problems():
    q = _q()
    n, k = 1000, 1088
    bases = [_mixed_base(n, k, BF16, seed=70 + i) for i in range(2)]
    _, sets = _adapter_sets(n, k, ([8, 16], [16, 8]), BF16, seed=90)
    x = make_act(32, k, seed=1)
    with pytest.raises(ValueError, match="same rank"):
        q.lora_linear4bit_group_multi(x, bases, sets, torch.zeros(32, dtype=torch.int32, device="cuda"))
