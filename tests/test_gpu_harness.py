"""GPU tests of the bench harness (caller-side scaffolding): fused RoPE / SwiGLU kernels vs their torch formulations,
one tiny Llama-QLoRA training step (fused kernel + fused LoRA step + checkpointing) vs the all-unfused variant, and the
harness kernels element by element against float64 (the seeded dropout bit for bit)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def H():
    assert torch.cuda.is_available()
    import harness.llama_qlora as H
    from harness import fused_ops

    fused_ops.build()
    assert fused_ops.available()
    return H


def test_rope_and_swiglu_match_torch(H):
    from harness import fused_ops

    torch.manual_seed(0)
    b, s, h, d = 2, 64, 4, 128
    cos, sin = H._rope_tables(s, d, 10000.0, "cuda")
    q = torch.randn(b, s, h, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(b, s, h, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    gq, gk = torch.randn_like(q), torch.randn_like(k)
    qo, ko = fused_ops.rope_qk(q, k, cos, sin)
    (qo * gq).sum().backward(retain_graph=True)
    (ko * gk).sum().backward()
    got = [qo.detach().float(), ko.detach().float(), q.grad.float(), k.grad.float()]
    q2, k2 = q.detach().clone().requires_grad_(True), k.detach().clone().requires_grad_(True)
    qr, kr = H._apply_rope(q2, cos, sin), H._apply_rope(k2, cos, sin)
    (qr * gq).sum().backward()
    (kr * gk).sum().backward()
    ref = [qr.detach().float(), kr.detach().float(), q2.grad.float(), k2.grad.float()]
    for a, r in zip(got, ref):
        assert (a - r).abs().max().item() <= 0.04 and ((a - r).norm() / r.norm()).item() < 5e-3
    g = torch.randn(4, 100, 704, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    u = torch.randn(4, 100, 704, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    dy = torch.randn_like(g)
    out = fused_ops.swiglu(g, u)
    out.backward(dy)
    g2, u2 = g.detach().clone().requires_grad_(True), u.detach().clone().requires_grad_(True)
    ref_out = torch.nn.functional.silu(g2) * u2
    ref_out.backward(dy)
    assert torch.equal(out, ref_out)   # forward reproduces torch's two roundings exactly
    for a, r in ((g.grad, g2.grad), (u.grad, u2.grad)):
        assert ((a.float() - r.float()).norm() / r.float().norm()).item() < 1e-2


@pytest.mark.parametrize("d", [512, 704, 4096, 8192, 16384])   # register-resident row kernel up to 8192, two-pass above
def test_rmsnorm_matches_torch(H, d):
    from harness import fused_ops

    torch.manual_seed(0)
    x = (torch.randn(3, 100, d, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
    w = (1 + 0.1 * torch.randn(d, device="cuda")).float()
    gy = torch.randn_like(x)
    y = fused_ops.rmsnorm(x, w, 1e-5)
    y.backward(gy)
    x2 = x.detach().float().requires_grad_(True)
    y2 = torch.nn.functional.rms_norm(x2, (d,), w, 1e-5)
    y2.backward(gy.float())
    assert ((y.float() - y2).norm() / y2.norm()).item() < 3e-3
    assert ((x.grad.float() - x2.grad).norm() / x2.grad.norm()).item() < 5e-3


def _tiny_step(H, fused, group, dropout=0.0, norm_out_fp32=False, seed_bump=1):
    shape = H.SHAPES["tiny"]
    ids, labels = H.synthetic_batch(shape, 256, seed=0)
    ids, labels = ids.cuda(), labels.cuda()
    H.GROUP_LINEARS = group
    torch.manual_seed(0)  # lora_A / embeddings / lm_head are initialised from the global RNG
    model = H.LlamaQLoRA(shape, torch.device("cuda"), lora_r=16, seed=7, lora_dropout=dropout, norm_out_fp32=norm_out_fp32).train()
    torch.manual_seed(1)
    for idx, m in enumerate(mm for mm in model.modules() if isinstance(mm, H.LoRALinear4bit)):
        m.fused = fused
        m.salt = idx             # the same call-site ids in every model built by these tests
        torch.nn.init.normal_(m.lora_B.weight, std=0.05)  # non-zero B so the LoRA path carries signal
    model.dropout_seed.add_(seed_bump)
    loss = model(ids, labels)
    loss.backward()
    H.GROUP_LINEARS = True
    return loss.item(), torch.cat([p.grad.float().flatten() for p in model.trainable_parameters()]), model


def test_tiny_model_step_fused_vs_unfused(H):
    """One tiny Llama-QLoRA training step built through HF's replace_with_bnb_linear: fused NF4 GEMM + fused LoRA step +
    grouped q/k/v / gate/up launches + caller-side fusions vs the all-unfused variant."""
    res = []
    for fused, group in ((True, True), (True, False), (False, False)):
        H.USE_FUSED_OPS = fused
        res.append(_tiny_step(H, fused, group)[:2])
    H.USE_FUSED_OPS = True
    losses = [r[0] for r in res]
    assert all(torch.isfinite(torch.tensor(losses)))
    for i in (0, 1):
        assert abs(losses[i] - losses[2]) < 2e-2 * abs(losses[2])
        cos = torch.nn.functional.cosine_similarity(res[i][1], res[2][1], dim=0).item()
        assert cos > 0.99, (i, cos)
    # grouped vs per-linear launches of the same fused kernels: near-identical gradients
    assert torch.nn.functional.cosine_similarity(res[0][1], res[1][1], dim=0).item() > 0.9995


def test_tiny_model_lora_dropout_fused_matches_unfused_same_mask(H):
    """--lora_dropout 0.1 (the recipe's setting): the seeded mask is a function of (seed tensor, call site, index), so the
    fused-grouped model, the fused per-linear model and the unfused (peft-form) model all see the SAME masks; the checkpoint
    recompute regenerates them.  A different seed gives different gradients."""
    base_loss, base_grad, _ = _tiny_step(H, False, False, dropout=0.1)
    for fused, group in ((True, True), (True, False)):
        loss, grad, _ = _tiny_step(H, fused, group, dropout=0.1)
        assert abs(loss - base_loss) < 2e-2 * abs(base_loss)
        assert torch.nn.functional.cosine_similarity(grad, base_grad, dim=0).item() > 0.99
    loss2, grad2, _ = _tiny_step(H, True, True, dropout=0.1, seed_bump=2)
    assert torch.nn.functional.cosine_similarity(grad2, base_grad, dim=0).item() < 0.9999
    l0, g0, _ = _tiny_step(H, True, True, dropout=0.0)
    assert torch.nn.functional.cosine_similarity(g0, base_grad, dim=0).item() < 0.9999   # dropout really changes the step


def test_seeded_dropout_statistics_and_determinism(H):
    from harness import fused_ops

    x = torch.ones(1 << 20, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    seed = torch.tensor(5, device="cuda", dtype=torch.int64)
    y = fused_ops.seeded_dropout(x, 0.1, seed, 3)
    keep = (y != 0).float().mean().item()
    assert abs(keep - 0.9) < 3e-3 and torch.allclose(y[y != 0].float(), torch.tensor(1 / 0.9).to(torch.bfloat16).float())
    assert torch.equal(fused_ops.seeded_dropout(x, 0.1, seed, 3), y)            # same (seed, salt): same mask
    assert not torch.equal(fused_ops.seeded_dropout(x, 0.1, seed, 4), y)        # another call site
    assert not torch.equal(fused_ops.seeded_dropout(x, 0.1, seed + 1, 3), y)    # another step
    y.backward(torch.ones_like(y))
    assert torch.equal(x.grad, y.detach())                                      # backward applies the same mask and scale


def test_tiny_model_fp32_norm_flow(H):
    """`norm_out_fp32=True`: the reference's dtype flow (fp32 norm outputs -> Linear4bit sees fp32, returns fp32).  Same
    values as the bf16-emitting norms up to the norm's own rounding, fused vs unfused agree."""
    l_f, g_f, _ = _tiny_step(H, True, True, norm_out_fp32=True)
    l_u, g_u, _ = _tiny_step(H, False, False, norm_out_fp32=True)
    l_b, g_b, _ = _tiny_step(H, True, True, norm_out_fp32=False)
    assert abs(l_f - l_u) < 2e-2 * abs(l_u) and abs(l_f - l_b) < 2e-2 * abs(l_b)
    assert torch.nn.functional.cosine_similarity(g_f, g_u, dim=0).item() > 0.99
    assert torch.nn.functional.cosine_similarity(g_f, g_b, dim=0).item() > 0.99


@pytest.mark.parametrize("d", [512, 4096, 8192])
def test_add_rmsnorm_matches_unfused(H, d):
    """Residual add + RMSNorm in one kernel (forward and backward) vs `x + delta` followed by the stand-alone norm op."""
    from harness import fused_ops

    torch.manual_seed(0)
    x = (torch.randn(2, 70, d, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
    dl = torch.randn(2, 70, d, device="cuda").to(torch.bfloat16).requires_grad_(True)
    w = (1 + 0.1 * torch.randn(d, device="cuda")).float()
    g_s, g_y = torch.randn_like(x), torch.randn_like(x)
    s, y = fused_ops.add_rmsnorm(x, dl, w, 1e-5)
    torch.autograd.backward([s, y], [g_s, g_y])
    x2, d2 = x.detach().clone().requires_grad_(True), dl.detach().clone().requires_grad_(True)
    s2 = x2 + d2
    y2 = fused_ops.rmsnorm(s2, w, 1e-5)
    torch.autograd.backward([s2, y2], [g_s, g_y])
    assert torch.equal(s, s2) and torch.equal(y, y2)
    for a, b in ((x.grad, x2.grad), (dl.grad, d2.grad)):
        assert ((a.float() - b.float()).norm() / b.float().norm()).item() < 4e-3   # one rounding instead of two


# ---------------------------------------------------------------------------------------------------------------------
# Element-wise checks against float64 computed from the same bf16 inputs.  The bound of every element is one bf16 ulp of
# the float64 result plus the kernel's fp32 roundings, scaled by the magnitudes of the terms they act on (`mag`): where a
# backward subtracts nearly equal terms, the fp32 error of those terms can exceed an ulp of the small difference.
# ---------------------------------------------------------------------------------------------------------------------
def _bf16_ulp(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |v| (float64; 0 where v is 0)."""
    _, e = torch.frexp(v.abs())
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), e - 8))


def _assert_elementwise(got, ref, mag, fp32_ulps, what):
    got = got.detach().double().cpu()
    tol = _bf16_ulp(ref) + fp32_ulps * 2.0 ** -24 * mag
    bad = (got - ref).abs() > tol
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {bad.nonzero()[0].tolist()}: "
                           f"{got[bad][0].item()} vs {ref[bad][0].item()} (tol {tol[bad][0].item():.3e})")


def _f64(t):
    return t.detach().double().cpu()


@pytest.mark.parametrize("n", [4096, 132 * 16 * 256 * 8 + 8 * 4099])   # the second runs past the kernel's grid-stride cap
def test_seeded_dropout_is_bit_exact(H, n):
    """The mask and scale of the seeded dropout, forward and backward, against tests/step_reference.py's restatement of the
    kernel's hash."""
    import step_reference as R
    from harness import fused_ops

    torch.manual_seed(11)
    x = torch.randn(n, device="cuda").to(torch.bfloat16).requires_grad_(True)
    gy = torch.randn(n, device="cuda").to(torch.bfloat16)
    for p in (0.0, 0.1, 0.5):
        scale = torch.tensor(1.0) / (1.0 - torch.tensor(p, dtype=torch.float32))   # the kernel's fp32 1 / (1 - p)
        for seed, salt in ((1, 1), (2, 1), (1, 2), (123456789, 77)):
            seed_dev = torch.tensor(seed, device="cuda", dtype=torch.int64)
            keep = torch.from_numpy(R.dropout_keep(n, p, seed, salt))
            x.grad = None
            y = fused_ops.seeded_dropout(x, p, seed_dev, salt)
            y.backward(gy)
            for out, src in ((y, x), (x.grad, gy)):
                want = torch.where(keep, (src.detach().float().cpu() * scale).to(torch.bfloat16), torch.zeros((), dtype=torch.bfloat16))
                assert torch.equal(out.detach().cpu(), want), (p, seed, salt)
            if p == 0.0:
                assert torch.equal(y, x)


def test_rope_tables_match_float64(H):
    """cos and sign-folded sin, [seq, 1, d] bf16: within one bf16 ulp of float64, plus the fp32 rounding of the angle
    (position x inverse frequency in fp32, as HF computes it)."""
    s, d, theta = 2048, 128, 10000.0
    cos, sin = H._rope_tables(s, d, theta, "cuda")
    assert cos.shape == (s, 1, d) and sin.shape == (s, 1, d)
    inv = 1.0 / theta ** (torch.arange(0, d, 2, dtype=torch.float64) / d)
    ang = torch.outer(torch.arange(s, dtype=torch.float64), inv)
    slack = 2.0 ** -22 * ang.repeat(1, 2)   # the fp32 angle: |error| <= ~2 ulp of it
    for got, want in ((cos, torch.cat((ang.cos(), ang.cos()), -1)), (sin, torch.cat((-ang.sin(), ang.sin()), -1))):
        assert ((_f64(got[:, 0]) - want).abs() <= _bf16_ulp(want) + slack).all()


def _rope64(x, cos, sin):
    half = x.shape[-1] // 2
    return x * cos + torch.cat((x[..., half:], x[..., :half]), -1) * sin


@pytest.mark.parametrize("d", [64, 128])
def test_rope_matches_float64(H, d):
    """Forward and backward (the kernel with sign -1) at batch 3 with more q heads than k heads (grouped-query attention),
    every element within one bf16 ulp of float64 from the same bf16 inputs and tables."""
    from harness import fused_ops

    torch.manual_seed(d)
    b, s, hq, hk = 3, 97, 8, 2
    cos, sin = H._rope_tables(s, d, 10000.0, "cuda")
    q = torch.randn(b, s, hq, d, device="cuda").to(torch.bfloat16).requires_grad_(True)
    k = torch.randn(b, s, hk, d, device="cuda").to(torch.bfloat16).requires_grad_(True)
    gq, gk = torch.randn_like(q), torch.randn_like(k)
    qo, ko = fused_ops.rope_qk(q, k, cos, sin)
    torch.autograd.backward([qo, ko], [gq, gk])
    c64, s64 = _f64(cos), _f64(sin)
    for x, g, out in ((q, gq, qo), (k, gk, ko)):
        x64 = _f64(x).requires_grad_(True)
        y64 = _rope64(x64, c64, s64)
        y64.backward(_f64(g))
        mag = _rope64(x64.detach().abs(), c64.abs(), s64.abs())
        _assert_elementwise(out, y64.detach(), mag, 4, f"rope fwd h={x.shape[2]}")
        gmag = _rope64(_f64(g).abs(), c64.abs(), s64.abs())   # the transpose mixes the same pairs
        _assert_elementwise(x.grad, x64.grad, gmag, 4, f"rope bwd h={x.shape[2]}")


def _rms64(x, w, eps):
    rstd = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    return x * rstd * w, rstd


def _rms_bwd_mag(x, w, g, rstd):
    """Magnitudes of the terms of dx = rstd (g w - x c), c = rstd^2 mean(g w x): what the fp32 roundings act on."""
    cmag = rstd * rstd * (g * w * x).abs().mean(-1, keepdim=True)
    return rstd * ((g * w).abs() + x.abs() * cmag)


NORM_DIMS = [2048, 2056, 4096, 4104, 8192, 8200]   # each side of the register-tile (2/4/8 vectors) and two-pass boundaries


@pytest.mark.parametrize("d", NORM_DIMS)
def test_rmsnorm_matches_float64(H, d):
    from harness import fused_ops

    torch.manual_seed(d)
    x = (torch.randn(3, 67, d, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)   # 201 rows
    w = (1 + 0.1 * torch.randn(d, device="cuda")).float()
    gy = torch.randn_like(x)
    y = fused_ops.rmsnorm(x, w, 1e-5)
    y.backward(gy)
    x64 = _f64(x).requires_grad_(True)
    w64, g64 = _f64(w), _f64(gy)
    y64, rstd = _rms64(x64, w64, 1e-5)
    y64.backward(g64)
    _assert_elementwise(y, y64.detach(), y64.detach().abs(), d / 4, f"rmsnorm fwd d={d}")
    _assert_elementwise(x.grad, x64.grad, _rms_bwd_mag(x64.detach(), w64, g64, rstd.detach()), d / 4, f"rmsnorm bwd d={d}")


@pytest.mark.parametrize("d", NORM_DIMS)
def test_add_rmsnorm_matches_float64(H, d):
    """The residual sum is torch's bf16 `x + delta` exactly; the norm of it and both input gradients (the residual-path
    gradient plus the norm's backward) within the element bound of float64."""
    from harness import fused_ops

    torch.manual_seed(d + 1)
    x = (torch.randn(3, 67, d, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
    dl = torch.randn(3, 67, d, device="cuda").to(torch.bfloat16).requires_grad_(True)
    w = (1 + 0.1 * torch.randn(d, device="cuda")).float()
    if d > 8192:   # one CTA holds the row in registers: 8192 is the widest row the fused form takes
        with pytest.raises(RuntimeError, match="failed"):
            fused_ops.add_rmsnorm(x, dl, w, 1e-5)
        return
    g_s, g_y = torch.randn_like(x), torch.randn_like(x)
    s, y = fused_ops.add_rmsnorm(x, dl, w, 1e-5)
    torch.autograd.backward([s, y], [g_s, g_y])
    assert torch.equal(s.cpu(), (x.detach().float() + dl.detach().float()).to(torch.bfloat16).cpu())
    s64 = _f64(s).requires_grad_(True)
    w64, gs64, gy64 = _f64(w), _f64(g_s), _f64(g_y)
    y64, rstd = _rms64(s64, w64, 1e-5)
    y64.backward(gy64)
    _assert_elementwise(y, y64.detach(), y64.detach().abs(), d / 4, f"add_rmsnorm fwd d={d}")
    want = gs64 + s64.grad
    mag = gs64.abs() + _rms_bwd_mag(s64.detach(), w64, gy64, rstd.detach())
    for grad in (x.grad, dl.grad):
        _assert_elementwise(grad, want, mag, d / 4, f"add_rmsnorm bwd d={d}")


def test_swiglu_backward_matches_float64(H):
    """d_gate = dy u s (1 + g (1 - s)) and d_up = dy g s, s = sigmoid(g), from the same bf16 inputs; the kernel's fast
    exponential is part of the fp32 term."""
    from harness import fused_ops

    torch.manual_seed(5)
    g = (torch.randn(3, 101, 704, device="cuda") * 3).to(torch.bfloat16).requires_grad_(True)
    u = torch.randn(3, 101, 704, device="cuda").to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn_like(g)
    fused_ops.swiglu(g, u).backward(dy)
    g64, u64, dy64 = _f64(g), _f64(u), _f64(dy)
    sg = torch.sigmoid(g64)
    dg = dy64 * u64 * sg * (1 + g64 * (1 - sg))
    du = dy64 * g64 * sg
    mag_g = (dy64 * u64).abs() * (sg + (g64 * sg * (1 - sg)).abs()) * (1 + g64.abs())   # __expf's error grows with |g|
    _assert_elementwise(g.grad, dg, mag_g, 16, "swiglu d_gate")
    _assert_elementwise(u.grad, du, du.abs() * (1 + g64.abs()), 16, "swiglu d_up")
