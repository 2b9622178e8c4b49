"""The dX launch of a checkpointed layer reads the bf16 weight copies its checkpoint recompute wrote.

At training token counts every Linear4bit call dequantizes its NF4 weights into a bf16 scratch that the TMA-fed GEMM reads
(the scratch path).  A forward that runs inside a backward (the recompute of a checkpointed layer) keeps that scratch for
the layer's dX launch, which then skips its own dequantize.  The copies are bit-exact, so every result stays the same: a
checkpointed step equals the plain step bit for bit, with non-reentrant and reentrant checkpointing, grouped and per-linear
launches, LoRA dropout and fp32 norm outputs, and under CUDA-graph replay.  A forward outside backward keeps no copy."""
import pytest
import torch
import torch.utils.checkpoint

from gpu_helpers import make_act, make_weight

pytestmark = pytest.mark.gpu


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
    """The attention backward and cuBLAS in their deterministic forms (as bench.py runs them), so that two runs of one step
    can be compared bit for bit."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev, prev_fill = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    yield
    torch.use_deterministic_algorithms(prev)
    torch.utils.deterministic.fill_uninitialized_memory = prev_fill


def _scratch_path_active():
    from qlora_b200 import _lib

    return _lib.load().qb200_nf4_linear_scratch_size(1, 1543, 256, 256, 0) > 0


def _reentrant_checkpoint(fn, *args, use_reentrant=False, preserve_rng_state=True):
    return torch.utils.checkpoint.checkpoint(fn, *args, use_reentrant=True, preserve_rng_state=preserve_rng_state)


def _tiny_model(H, seq, ckpt, group=True, dropout=0.0, norm_out_fp32=False):
    shape = H.SHAPES["tiny"]
    ids, labels = H.synthetic_batch(shape, seq, seed=3)
    torch.manual_seed(0)
    model = H.LlamaQLoRA(shape, torch.device("cuda"), lora_r=16, seed=7, lora_dropout=dropout, norm_out_fp32=norm_out_fp32,
                         grad_checkpointing=ckpt != "none").train()
    torch.manual_seed(1)
    for idx, m in enumerate(mm for mm in model.modules() if isinstance(mm, H.LoRALinear4bit)):
        m.salt = idx
        torch.nn.init.normal_(m.lora_B.weight, std=0.05)   # non-zero B: the LoRA terms of dX carry signal
    model.dropout_seed.add_(1)
    model.test_group = group
    return model, ids.cuda(), labels.cuda()


def _step(H, model, ids, labels, ckpt, monkeypatch):
    """One forward + backward; returns (loss, every adapter gradient flattened)."""
    with monkeypatch.context() as mp:
        mp.setattr(H, "GROUP_LINEARS", model.test_group)
        if ckpt == "reentrant":
            mp.setattr(H, "checkpoint", _reentrant_checkpoint)
        for p in model.trainable_parameters():
            p.grad = None
        loss = model(ids, labels)
        loss.backward()
    return loss.detach().clone(), torch.cat([p.grad.float().flatten() for p in model.trainable_parameters()])


CONFIGS = {"grouped": {}, "per_linear": {"group": False}, "dropout": {"dropout": 0.1}, "norm_out_fp32": {"norm_out_fp32": True}}


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("ckpt", ["non_reentrant", "reentrant"])
@pytest.mark.parametrize("seq", [1543, 2048])
def test_checkpointed_step_equals_plain_step_bitwise(H, deterministic, monkeypatch, seq, ckpt, config):
    assert _scratch_path_active()
    plain = _step(H, *_tiny_model(H, seq, "none", **CONFIGS[config]), "none", monkeypatch)
    ckpted = _step(H, *_tiny_model(H, seq, ckpt, **CONFIGS[config]), ckpt, monkeypatch)
    assert torch.isfinite(plain[0])
    assert torch.equal(plain[0], ckpted[0]) and torch.equal(plain[1], ckpted[1])


@pytest.mark.parametrize("seq", [1543, 2048])
def test_checkpointed_step_replays_under_cuda_graphs(H, deterministic, monkeypatch, seq):
    model, ids, labels = _tiny_model(H, seq, "non_reentrant")
    eager = _step(H, model, ids, labels, "non_reentrant", monkeypatch)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _step(H, model, ids, labels, "non_reentrant", monkeypatch)
    torch.cuda.current_stream().wait_stream(side)
    for p in model.trainable_parameters():
        p.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="thread_local"):
        loss = model(ids, labels)
        loss.backward()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    grads = torch.cat([p.grad.float().flatten() for p in model.trainable_parameters()])
    assert torch.equal(loss, eager[0]) and torch.equal(grads, eager[1])


@pytest.mark.parametrize("group", [True, False])
@pytest.mark.parametrize("ckpt", ["non_reentrant", "reentrant"])
def test_checkpointed_step_dequantizes_each_weight_twice(H, monkeypatch, ckpt, group):
    """Forward and recompute dequantize every weight, the dX launches none.  Before the recompute's copies were reused, a
    checkpointed step dequantized each weight 3 times."""
    import qlora_b200.functional as QF

    model, ids, labels = _tiny_model(H, 2048, ckpt, group=group)
    _step(H, model, ids, labels, ckpt, monkeypatch)   # warm-up
    QF.LAUNCH_COUNTER[0] = 0
    QF.EVENT_LOG = []   # one entry per GEMM launch
    try:
        _step(H, model, ids, labels, ckpt, monkeypatch)
        gemms = len(QF.EVENT_LOG)
    finally:
        QF.EVENT_LOG = None
    layers = H.SHAPES["tiny"].layers
    assert gemms == 3 * (4 if group else 7) * layers
    assert QF.LAUNCH_COUNTER[0] - gemms == 2 * 7 * layers


def _linear4bit(n, k, seed):
    import qlora_b200 as q

    lin = q.nn.Linear4bit(k, n, bias=False, compute_dtype=torch.bfloat16, compress_statistics=True, quant_type="nf4")
    lin.weight = q.nn.Params4bit(make_weight(n, k, seed, device="cpu"), requires_grad=False, compress_statistics=True,
                                 quant_type="nf4", module=lin)
    return lin.to("cuda")


def test_plain_linear4bit_reuses_the_recompute_copy(deterministic):
    """A Linear4bit without adapters (peft targeting only q/v leaves the others plain) under checkpointing: same input
    gradient as without, and its dX launch dequantizes nothing."""
    import qlora_b200.functional as QF

    lin = _linear4bit(1024, 512, seed=5)
    x0 = make_act(2048, 512, seed=6)
    dy = make_act(2048, 1024, seed=7)
    grads, dequants = [], []
    for ckpt in (False, True):
        x = x0.clone().requires_grad_(True)
        QF.LAUNCH_COUNTER[0] = 0
        y = torch.utils.checkpoint.checkpoint(lin, x, use_reentrant=False) if ckpt else lin(x)
        y.backward(dy)
        grads.append(x.grad)
        dequants.append(QF.LAUNCH_COUNTER[0] - (3 if ckpt else 2))   # minus the GEMM launches
    assert torch.equal(grads[0], grads[1]) and dequants == [2, 2]


# 7B grouped shapes (q/k/v, o, gate/up, down: nprob, N, K) at 2048 tokens, and a ragged one at 1543
SHAPES = [(3, 4096, 4096, 2048), (1, 4096, 4096, 2048), (2, 11008, 4096, 2048), (1, 4096, 11008, 2048), (2, 4104, 4160, 1543)]


def _problems(nprob, n, k, m, r=64, seed=0):
    import qlora_b200.functional as QF

    ps, qss = zip(*[QF.quantize_4bit(make_weight(n, k, seed=seed + i), compress_statistics=True, quant_type="nf4")
                    for i in range(nprob)])
    return dict(ps=[p.t() for p in ps], qss=list(qss), x=make_act(m, k, seed=seed + 10),
                us=[make_act(m, r, seed=seed + 20 + i) for i in range(nprob)], vs=[make_weight(n, r, seed=seed + 30 + i) for i in range(nprob)],
                dys=[make_act(m, n, seed=seed + 40 + i) for i in range(nprob)], gs=[make_act(m, r, seed=seed + 50 + i) for i in range(nprob)],
                as_=[make_weight(r, k, seed=seed + 60 + i) for i in range(nprob)])


@pytest.mark.parametrize("nprob,n,k,m", SHAPES)
def test_dx_with_reused_scratch_equals_fresh_dx(nprob, n, k, m):
    import qlora_b200.functional as QF

    d = _problems(nprob, n, k, m)
    ys, scratch = QF.nf4_linear_group(False, [d["x"]] * nprob, d["ps"], d["qss"], us=d["us"], vs=d["vs"], return_scratch=True)
    assert scratch is not None and scratch.numel() == nprob * n * k * 2
    assert all(torch.equal(a, b) for a, b in zip(ys, QF.nf4_linear_group(False, [d["x"]] * nprob, d["ps"], d["qss"], us=d["us"], vs=d["vs"])))
    QF.LAUNCH_COUNTER[0] = 0
    fresh = QF.nf4_linear_group(True, d["dys"], d["ps"], d["qss"], us=d["gs"], vs=d["as_"])
    assert QF.LAUNCH_COUNTER[0] == 1 + nprob
    QF.LAUNCH_COUNTER[0] = 0
    reused, left = QF.nf4_linear_group(True, d["dys"], d["ps"], d["qss"], us=d["gs"], vs=d["as_"], w_scratch=scratch,
                                       return_scratch=True)
    assert QF.LAUNCH_COUNTER[0] == 1 and left is scratch
    assert torch.equal(fresh, reused)
    # without LoRA operands (the dX of a dropout step)
    plain = QF.nf4_linear_group(True, d["dys"], d["ps"], d["qss"])
    assert torch.equal(plain, QF.nf4_linear_group(True, d["dys"], d["ps"], d["qss"], w_scratch=scratch))


def test_reused_scratch_is_what_the_gemm_reads():
    """A dX told that the workspace holds its weights runs no dequantize: given another weight's copy, it computes with
    that weight."""
    import qlora_b200.functional as QF

    a, b = _problems(1, 4096, 4096, 2048, seed=0), _problems(1, 4096, 4096, 2048, seed=100)
    _, scratch_b = QF.nf4_linear_group(False, [b["x"]], b["ps"], b["qss"], return_scratch=True)
    want = QF.nf4_linear_group(True, a["dys"], b["ps"], b["qss"])
    got = QF.nf4_linear_group(True, a["dys"], a["ps"], a["qss"], w_scratch=scratch_b)
    assert torch.equal(got, want) and not torch.equal(got, QF.nf4_linear_group(True, a["dys"], a["ps"], a["qss"]))


def test_calls_off_the_scratch_path_leave_no_scratch():
    """A forward whose bf16 output pitch is not 16-byte aligned runs the fused kernel: it reports no scratch and ignores
    one passed in.  A scratch too short for the call is refused before any launch."""
    import qlora_b200.functional as QF
    from qlora_b200._lib import Qb200Error

    nprob, n, k, m = 2, 4096, 4096, 2048
    d = _problems(nprob, n, k, m)
    _, scratch = QF.nf4_linear_group(False, [d["x"]] * nprob, d["ps"], d["qss"], return_scratch=True)
    bufs = [torch.empty((m, n + 4), dtype=torch.bfloat16, device="cuda") for _ in range(nprob)]
    QF.LAUNCH_COUNTER[0] = 0
    ys, left = QF.nf4_linear_group(False, [d["x"]] * nprob, d["ps"], d["qss"], outs=[t[:, :n] for t in bufs], return_scratch=True)
    assert left is None and QF.LAUNCH_COUNTER[0] == 1
    ref = QF.nf4_linear_group(False, [d["x"]] * nprob, d["ps"], d["qss"])
    assert all(torch.equal(a, b) for a, b in zip(ys, ref))
    bufs2 = [torch.empty((m, n + 4), dtype=torch.bfloat16, device="cuda") for _ in range(nprob)]
    ys2 = QF.nf4_linear_group(False, [d["x"]] * nprob, d["ps"], d["qss"], outs=[t[:, :n] for t in bufs2], w_scratch=scratch)
    assert all(torch.equal(a, b) for a, b in zip(ys2, ref))
    with pytest.raises(Qb200Error, match="invalid argument"):
        QF.nf4_linear_group(True, d["dys"], d["ps"], d["qss"], w_scratch=scratch[: scratch.numel() // 2])


def test_forward_outside_backward_keeps_no_copy():
    """A non-checkpointed forward (gate/up at the 7B shape, 2048 tokens) holds its outputs and small saved tensors, not the
    180 MB of bf16 weights."""
    from qlora_b200 import lora

    n, k, m, r = 11008, 4096, 2048, 64
    bases = [_linear4bit(n, k, seed=20 + i) for i in range(2)]
    a_s = [torch.nn.Parameter(make_weight(r, k, seed=30 + i)) for i in range(2)]
    b_s = [torch.nn.Parameter(make_weight(n, r, seed=40 + i)) for i in range(2)]
    x = make_act(m, k, seed=50).requires_grad_(True)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    ys = lora.lora_linear4bit_group(x, bases, a_s, b_s, 0.25)
    torch.cuda.synchronize()
    grew = torch.cuda.memory_allocated() - before
    scratch_bytes = 2 * n * k * 2
    assert sum(y.numel() * y.element_size() for y in ys) <= grew < scratch_bytes
