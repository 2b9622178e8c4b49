"""CPU checks of the float64 step restatement (tests/step_reference.py): its dropout masks against a pure-Python integer
restatement of the kernel's hash, and its adapter gradients against finite differences on a random model of the tiny
harness structure."""
import numpy as np
import pytest
import torch

import step_reference as R

_M64 = (1 << 64) - 1


def _splitmix64(z):
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def _kept_py(i, thr16, seed, salt):
    """dropout_kernel for element i, in its own terms: vector i // 8, words rr[0..3] from r0, r1, lo / hi 16-bit lanes."""
    key = _splitmix64((seed * 0xD1342543DE82EF95 + salt) & _M64)
    vec, j = divmod(i, 8)
    r0, r1 = _splitmix64(key ^ (2 * vec)), _splitmix64(key ^ (2 * vec + 1))
    rr = (r0 & 0xFFFFFFFF, r0 >> 32, r1 & 0xFFFFFFFF, r1 >> 32)[j // 2]
    lane = rr & 0xFFFF if j % 2 == 0 else rr >> 16
    return lane >= thr16


def test_dropout_thresholds():
    assert [R.dropout_threshold(p) for p in (0.0, 0.1, 0.5)] == [0, 6554, 32768]


@pytest.mark.parametrize("p,seed,salt", [(0.1, 1, 1), (0.1, 2, 1), (0.5, 7, 13), (0.1, 1 << 40, 3), (0.3, 12345, 1 << 33)])
def test_numpy_mask_matches_integer_hash(p, seed, salt):
    n = 4096
    keep = R.dropout_keep(n, p, seed, salt)
    thr = R.dropout_threshold(p)
    assert keep.tolist() == [_kept_py(i, thr, seed, salt) for i in range(n)]
    far = 5_000_000 - 8   # past the kernel's grid-stride cap of 132 * 16 * 256 vectors of 8
    assert R.dropout_keep(far + 8, p, seed, salt)[far:].tolist() == [_kept_py(far + j, thr, seed, salt) for j in range(8)]
    assert abs(keep.mean() - (1 - p)) < 0.03
    assert not np.array_equal(keep, R.dropout_keep(n, p, seed, salt + 1))
    assert R.dropout_keep(n, 0.0, seed, salt).all()


def _random_model(seq, p, seed=0, hidden=64, inter=96, layers=2, heads=4, vocab=48):
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape, std=0.02):
        return torch.randn(*shape, generator=g, dtype=torch.float64) * std

    d = hidden // heads
    inv = 1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float64) / d))
    fr = torch.outer(torch.arange(seq, dtype=torch.float64), inv)
    weights, salts = {}, {}
    for li in range(layers):
        for n in R.LINEARS:
            out_f, in_f = {"gate_proj": (inter, hidden), "up_proj": (inter, hidden), "down_proj": (hidden, inter)}.get(n, (hidden, hidden))
            weights[(li, n)] = rnd(out_f, in_f, std=0.1)
            salts[(li, n)] = 1 + len(salts)
    model = R.RefModel(weights=weights, norms={(li, k): 1 + rnd(hidden, std=0.1) for li in range(layers) for k in ("input", "post")},
                       final_norm=1 + rnd(hidden, std=0.1), embed=rnd(vocab, hidden, std=1.0), lm_head=rnd(vocab, hidden, std=0.3),
                       cos=torch.cat((fr.cos(), fr.cos()), -1), sin=torch.cat((-fr.sin(), fr.sin()), -1), heads=heads, eps=1e-5,
                       scaling=0.25, p=p, salts=salts)
    adapters = {}
    for (li, n), w in weights.items():
        adapters[R.adapter_name(li, n, "A")] = rnd(8, w.shape[1], std=0.1)
        adapters[R.adapter_name(li, n, "B")] = rnd(w.shape[0], 8, std=0.1)
    ids = torch.randint(0, vocab, (1, seq), generator=g)
    labels = ids.clone()
    labels[:, :5] = -100
    return model, adapters, ids, labels


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_gradients_match_finite_differences(p):
    model, adapters, ids, labels = _random_model(40, p)
    loss, grads = R.micro_step(model, adapters, ids, labels, seed=3)
    assert np.isfinite(loss) and set(grads) == set(adapters)
    g = torch.Generator().manual_seed(1)
    for name in (R.adapter_name(0, "q_proj", "A"), R.adapter_name(1, "down_proj", "B"), R.adapter_name(0, "k_proj", "B")):
        direction = torch.randn(adapters[name].shape, generator=g, dtype=torch.float64)
        h = 1e-5
        plus = dict(adapters, **{name: adapters[name] + h * direction})
        minus = dict(adapters, **{name: adapters[name] - h * direction})
        fd = (float(R.forward(model, plus, ids, labels, 3)) - float(R.forward(model, minus, ids, labels, 3))) / (2 * h)
        an = float((grads[name] * direction).sum())
        assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-3), (name, fd, an)


def test_zero_b_gives_zero_da_and_dropout_changes_the_step():
    model, adapters, ids, labels = _random_model(24, 0.1)
    zero_b = {n: (torch.zeros_like(t) if n.endswith("lora_B.weight") else t) for n, t in adapters.items()}
    _, grads = R.micro_step(model, zero_b, ids, labels, seed=3)
    assert all(not grads[n].any() for n in grads if n.endswith("lora_A.weight"))
    assert all(grads[n].abs().sum() > 0 for n in grads if n.endswith("lora_B.weight"))
    l3, g3 = R.micro_step(model, adapters, ids, labels, seed=3)
    l4, g4 = R.micro_step(model, adapters, ids, labels, seed=4)
    name = R.adapter_name(0, "v_proj", "A")
    assert not torch.equal(g3[name], g4[name])
