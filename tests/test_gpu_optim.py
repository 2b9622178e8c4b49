"""GPU parity for the 32-bit (paged) AdamW of SURVEY.md 8f-3 vs the oracle's restatement of upstream's update rule."""
import numpy as np
import pytest
import torch

from oracle import nf4_oracle as o

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("paged", [False, True])
def test_adamw32bit_matches_oracle(dtype, paged):
    import qlora_b200 as q

    torch.manual_seed(0)
    n = 64 * 1000 + 37
    p0 = (torch.randn(n) * 0.1).to(dtype)
    hp = dict(lr=2e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    p = torch.nn.Parameter(p0.clone().cuda())
    opt = q.optim.AdamW([p], is_paged=paged, **hp)
    pr = p0.float().numpy().copy()
    m = np.zeros(n, np.float32)
    v = np.zeros(n, np.float32)
    for step in range(1, 4):
        g = (torch.randn(n) * 0.01).to(dtype)
        p.grad = g.cuda()
        opt.step()
        pr, m, v = o.adamw32bit_step(pr, g.float().numpy(), m, v, hp["lr"], *hp["betas"], hp["eps"], hp["weight_decay"], step)
        pr = torch.from_numpy(pr).to(dtype).float().numpy()  # the parameter is stored in `dtype` between steps
        st = opt.state[p]
        assert np.allclose(st["state1"].cpu().numpy(), m, rtol=1e-6, atol=1e-12)
        assert np.allclose(st["state2"].cpu().numpy(), v, rtol=1e-6, atol=1e-18)
        got = p.detach().float().cpu().numpy()
        if dtype == torch.float32:
            assert np.allclose(got, pr, rtol=2e-6, atol=1e-9)
        else:  # identical up to one rounding step of the storage dtype
            ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
            assert np.all(np.abs(got - pr) <= ulp * np.maximum(np.abs(pr), 1e-3) * 1.01)
    assert opt.state[p]["step"] == 3


def test_paged_equals_resident_and_torch():
    import qlora_b200 as q

    torch.manual_seed(1)
    w = torch.randn(256, 64, device="cuda")
    params = [torch.nn.Parameter(w.clone()) for _ in range(3)]
    opts = [q.optim.PagedAdamW32bit([params[0]], lr=1e-3, weight_decay=0.0), q.optim.AdamW32bit([params[1]], lr=1e-3, weight_decay=0.0),
            torch.optim.AdamW([params[2]], lr=1e-3, weight_decay=0.0)]
    for _ in range(5):
        g = torch.randn_like(w)
        for prm, opt in zip(params, opts):
            prm.grad = g.clone()
            opt.step()
    assert torch.equal(params[0], params[1])                       # paged state changes nothing numerically
    assert torch.allclose(params[0], params[2], rtol=1e-5, atol=1e-7)  # same optimizer as torch's AdamW
    st = opts[0].state[params[0]]
    assert st["state1"].is_cuda and st["state1"].dtype == torch.float32
    assert set(st) == {"step", "state1", "state2"} and all(torch.is_tensor(v) for v in st.values())  # tensors only (ADVICE r1)
    opts[0]._paged[id(params[0])][0].prefetch(False)   # evict to host and touch again from the GPU: unified memory round trip
    torch.cuda.synchronize()
    assert torch.isfinite(st["state1"]).all()


@pytest.mark.parametrize("paged", [False, True])
def test_state_dict_save_load_step_roundtrip(paged, tmp_path):
    """optimizer.pt as HF Trainer writes it: torch.save(state_dict) -> fresh optimizer -> load_state_dict -> step.
    The file holds tensors only (weights_only load works), loaded paged moments get fresh unified-memory homes, and the
    resumed run continues bit-identically to the uninterrupted one."""
    import qlora_b200 as q

    torch.manual_seed(2)
    w = torch.randn(300, 33, device="cuda", dtype=torch.bfloat16)
    grads = [torch.randn_like(w) * 0.01 for _ in range(4)]
    hp = dict(lr=1e-3, weight_decay=0.01, is_paged=paged)
    pa = torch.nn.Parameter(w.clone())
    oa = q.optim.AdamW([pa], **hp)
    for g in grads:
        pa.grad = g.clone()
        oa.step()
    pb = torch.nn.Parameter(w.clone())
    ob = q.optim.AdamW([pb], **hp)
    for g in grads[:2]:
        pb.grad = g.clone()
        ob.step()
    f = tmp_path / "optimizer.pt"
    torch.save(ob.state_dict(), f)
    w_mid = pb.detach().clone()
    del ob
    pc = torch.nn.Parameter(w_mid)
    oc = q.optim.AdamW([pc], **hp)
    oc.load_state_dict(torch.load(f, weights_only=True))
    if paged:
        assert id(pc) in oc._paged and oc.state[pc]["state1"].data_ptr() == oc._paged[id(pc)][0].ptr
    for g in grads[2:]:
        pc.grad = g.clone()
        oc.step()
    assert torch.equal(pc, pa)
    assert float(oc.state[pc]["step"]) == 4


def test_capturable_step_in_cuda_graph_matches_eager():
    """`capturable=True`: step count and clip coefficient are device scalars -> the update is captured once and replayed."""
    import qlora_b200 as q

    torch.manual_seed(3)
    w = torch.randn(4096, 17, device="cuda", dtype=torch.bfloat16)
    grads = [torch.randn_like(w) * 0.02 for _ in range(5)]
    scales = [1.0, 0.5, 0.25, 1.0, 0.125]
    pe = torch.nn.Parameter(w.clone())
    oe = q.optim.PagedAdamW32bit([pe], lr=2e-4, weight_decay=0.0)
    for g, sc in zip(grads, scales):
        pe.grad = (g.float() * sc).to(torch.bfloat16)   # power-of-two scales: exact in bf16
        oe.step()
    pg = torch.nn.Parameter(w.clone())
    og = q.optim.PagedAdamW32bit([pg], lr=2e-4, weight_decay=0.0, capturable=True)
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
    og.state[pg]["state1"].zero_()
    og.state[pg]["state2"].zero_()
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
    assert torch.equal(pg, pe)


def test_step_flat_equals_per_parameter_steps():
    """`step_flat`: all parameters are views into one flat buffer (as are their gradients) and ONE launch updates them —
    bit-identical to per-parameter `step()` calls, clip coefficient included."""
    import qlora_b200 as q

    torch.manual_seed(4)
    shapes = [(64, 40), (40, 64), (16, 128)]
    n = sum(a * b for a, b in shapes)
    flat_p = (torch.randn(n, device="cuda") * 0.1).to(torch.bfloat16)
    flat_g = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    ref_params = []
    params = []
    off = 0
    for a, b in shapes:
        p = torch.nn.Parameter(flat_p[off:off + a * b].view(a, b))
        p.grad = flat_g[off:off + a * b].view(a, b)
        params.append(p)
        ref_params.append(torch.nn.Parameter(p.detach().clone()))
        off += a * b
    opt = q.optim.PagedAdamW32bit(params, lr=1e-3, weight_decay=0.0, capturable=True)
    ref = q.optim.AdamW32bit(ref_params, lr=1e-3, weight_decay=0.0)
    scale = torch.ones((), device="cuda")
    for step, sc in enumerate([1.0, 0.5, 0.25]):
        g = torch.randn(n, device="cuda") * 0.02
        flat_g.copy_(g.to(torch.bfloat16))
        scale.fill_(sc)
        off = 0
        for rp, (a, b) in zip(ref_params, shapes):
            rp.grad = (flat_g[off:off + a * b].float() * sc).to(torch.bfloat16).view(a, b).clone()
            off += a * b
        opt.step_flat(flat_p, flat_g, grad_scale=scale)
        ref.step()
        for p, rp in zip(params, ref_params):
            assert torch.equal(p, rp), step
    assert float(opt._step_dev.item()) == 3


def _flat_views(flat, shapes):
    params, off = [], 0
    for a, b in shapes:
        params.append(torch.nn.Parameter(flat[off:off + a * b].view(a, b)))
        off += a * b
    return params


@pytest.mark.parametrize("paged", [False, True])
def test_step_flat_state_dict_resumes_bitwise(paged, tmp_path):
    """optimizer.pt written after `step_flat` steps (the benchmarked configuration) holds the flat moments as per-parameter
    slices and the device-side step count: a fresh optimizer loaded from it continues bit-identically to the uninterrupted
    run.  The parameters are laid out in the flat buffer in another order than the optimizer lists them."""
    import qlora_b200 as q

    torch.manual_seed(5)
    shapes = [(64, 40), (40, 64), (16, 128)]
    n = sum(a * b for a, b in shapes)
    w = (torch.randn(n, device="cuda") * 0.05).to(torch.bfloat16)
    grads = [(torch.randn(n, device="cuda") * 0.01).to(torch.bfloat16) for _ in range(4)]
    scales = [1.0, 0.5, 0.25, 1.0]
    hp = dict(lr=1e-3, weight_decay=0.01, capturable=True, is_paged=paged)

    def run(flat_p, opt, steps):
        flat_g = torch.empty_like(flat_p)
        scale = torch.ones((), device="cuda")
        for g, sc in steps:
            flat_g.copy_(g)
            scale.fill_(sc)
            opt.step_flat(flat_p, flat_g, grad_scale=scale)

    flat_a = w.clone()
    pa = _flat_views(flat_a, shapes)
    run(flat_a, q.optim.AdamW(pa[::-1], **hp), list(zip(grads, scales)))
    flat_b = w.clone()
    pb = _flat_views(flat_b, shapes)
    ob = q.optim.AdamW(pb[::-1], **hp)
    run(flat_b, ob, list(zip(grads, scales))[:2])
    sd = ob.state_dict()
    assert sorted(sd["state"]) == [0, 1, 2] and all(float(st["step"]) == 2 for st in sd["state"].values())
    f = tmp_path / "optimizer.pt"
    torch.save(sd, f)
    flat_c = flat_b.clone()
    del ob, sd
    pc = _flat_views(flat_c, shapes)
    oc = q.optim.AdamW(pc[::-1], **hp)
    oc.load_state_dict(torch.load(f, weights_only=True))
    run(flat_c, oc, list(zip(grads, scales))[2:])
    assert torch.equal(flat_c, flat_a)
    assert float(oc._step_dev.item()) == 4
    if paged:
        assert oc._paged[id(oc._flat_key)][0].ptr == oc._flat[0].data_ptr()
    m_c, v_c = oc._flat
    assert all(torch.equal(st["state1"], m_c[off:off + p.numel()]) for st, p, off in
               zip(oc.state_dict()["state"].values(), oc.param_groups[0]["params"], oc._flat_offsets))
    assert torch.isfinite(v_c).all()
