"""Functional LM-MA-ES off the kernels: constants, validation, the float64 torch path against the paper-form oracle
(oracle/functional_lmmaes_oracle.py), recovery, item independence, the "max" sense, and the ABI return codes."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200.algorithms.functional import lmmaes, lmmaes_ask, lmmaes_tell, restarts
from evotorch_b200.algorithms.functional import funclmmaes as L
from oracle import functional_lmmaes_oracle as O

F64 = torch.float64


def _item(state, name, b=0):
    """Field `name` of item b of a torch state (any batch shape) as numpy."""
    t = getattr(state, name)
    core = {"center": 1, "sigma": 0, "p_sigma": 1, "M": 2, "G": 2}[name]
    return t.reshape((-1,) + tuple(t.shape[t.ndim - core:]))[b].numpy()


def _oracle_state(state, b=0):
    """The oracle's dict of item b of a torch state."""
    hp = state.hyperparameters
    s = O.init(_item(state, "center", b), float(_item(state, "sigma", b)), hp.popsize, hp.num_vectors, state.maximize)
    s.update(p_sigma=_item(state, "p_sigma", b).copy(), M=_item(state, "M", b).copy(), t=state.generation)
    return s


def _close(a, b, rtol=1e-12):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(np.abs(b).max(), 1e-300)
    assert np.abs(a - b).max() <= rtol * scale, (np.abs(a - b).max(), scale)


def _check_state(state, s, b=0, rtol=1e-12):
    _close(_item(state, "center", b), s["y"], rtol)
    _close(_item(state, "sigma", b), s["sigma"], rtol)
    _close(_item(state, "p_sigma", b), s["p_sigma"], rtol)
    _close(_item(state, "M", b), s["M"], rtol)
    _close(_item(state, "G", b), s["M"] @ s["M"].T, rtol)
    assert state.generation == s["t"]


@pytest.mark.parametrize("d", [5, 33, 100, 1000, 100003])
def test_constants(d):
    lam = 4 + int(math.floor(3 * math.log(d)))
    if d <= 2 * lam:
        with pytest.raises(ValueError, match=str(2 * lam + 1)):
            L.lmmaes_hyperparameters(d)
        return
    hp = L.lmmaes_hyperparameters(d, dtype=F64)
    mu = lam // 2
    raw = [math.log(mu + 0.5) - math.log(i) for i in range(1, mu + 1)]
    w = [r / sum(raw) for r in raw]
    assert hp.popsize == lam and hp.mu == mu and hp.num_vectors == lam
    np.testing.assert_allclose(hp.weights[:mu].numpy(), w, rtol=1e-15)
    assert torch.all(hp.weights[mu:] == 0)
    assert hp.mu_eff == pytest.approx(1 / sum(x * x for x in w), rel=1e-15)
    assert hp.c_sigma == pytest.approx(2 * lam / d, rel=1e-15)
    for j in range(1, lam + 1):
        assert hp.c_d[j - 1] == pytest.approx(1 / (1.5 ** (j - 1) * d), rel=1e-15)
        assert hp.c_c[j - 1] == pytest.approx(lam / (4 ** (j - 1) * d), rel=1e-15)
    hp2 = L.lmmaes_hyperparameters(d, popsize=7, num_vectors=3)
    assert hp2.popsize == 7 and hp2.mu == 3 and len(hp2.c_d) == 3


def test_validation():
    x0 = torch.zeros(40, dtype=F64)
    with pytest.raises(ValueError, match="objective_sense"):
        lmmaes(center_init=x0, stdev_init=1.0, objective_sense="minimize")
    with pytest.raises(ValueError, match="popsize"):
        lmmaes(center_init=x0, stdev_init=1.0, objective_sense="min", popsize=1)
    with pytest.raises(ValueError, match="num_vectors"):
        lmmaes(center_init=x0, stdev_init=1.0, objective_sense="min", num_vectors=0)
    with pytest.raises(ValueError, match="at least 41"):
        lmmaes(center_init=x0, stdev_init=1.0, objective_sense="min", popsize=20)
    with pytest.raises(TypeError, match="CMAESState or a SepCMAESState"):
        restarts(lmmaes(center_init=x0, stdev_init=1.0, objective_sense="min"), lb=-1.0, ub=1.0)
    s = lmmaes(center_init=x0, stdev_init=1.0, objective_sense="min")
    x = lmmaes_ask(s)
    with pytest.raises(ValueError, match="values"):
        lmmaes_tell(s, x[:-1], torch.zeros(s.popsize - 1, dtype=F64))
    with pytest.raises(ValueError, match="evals"):
        lmmaes_tell(s, x, torch.zeros(s.popsize + 1, dtype=F64))


def _run_against_oracle(d, gens, popsize=None, num_vectors=None, maximize=False, seed=0, inject=False):
    g = torch.Generator().manual_seed(seed)
    center = torch.randn(d, generator=g, dtype=F64)
    state = lmmaes(center_init=center, stdev_init=0.7, objective_sense="max" if maximize else "min", popsize=popsize, num_vectors=num_vectors)
    s = _oracle_state(state)
    A = torch.randn(d, d, generator=g, dtype=F64) / math.sqrt(d)
    ks = set()
    for _ in range(gens):
        ks.add(min(state.generation, state.num_vectors))
        z = torch.randn(1, state.popsize, d, generator=g, dtype=F64)
        x = L._ask_torch(state, z)[0]
        _close(x.numpy(), O.ask(s, z[0].numpy()))
        if inject:  # repaired / injected solutions: any values are legal
            x = x.clone()
            x[0] = torch.randn(d, generator=g, dtype=F64)
            x[1] = torch.clamp(x[1], -0.5, 0.5)
        f = ((x @ A.T) ** 2).sum(-1)
        state = lmmaes_tell(state, x, f)
        s = O.tell(s, x.numpy(), f.numpy())
        _check_state(state, s, rtol=1e-11)
    return ks


@pytest.mark.parametrize("d, popsize, num_vectors, gens", [(64, None, None, 30), (33, 7, 3, 12), (200, 9, 5, 8)])
def test_against_oracle(d, popsize, num_vectors, gens):
    ks = _run_against_oracle(d, gens, popsize, num_vectors)
    m = num_vectors or L.lmmaes_hyperparameters(d).num_vectors
    assert 0 in ks and m in ks and any(0 < k < m for k in ks)


def test_injected_values_against_oracle():
    _run_against_oracle(50, 12, 8, 4, inject=True, seed=3)


def test_maximize_against_oracle():
    _run_against_oracle(40, 10, 6, 3, maximize=True, seed=5)


def test_one_tell_of_asked_values():
    state = lmmaes(center_init=torch.ones(30, dtype=F64), stdev_init=1.5, objective_sense="min", popsize=6, num_vectors=2)
    s = _oracle_state(state)
    x = lmmaes_ask(state)
    f = (x * x).sum(-1)
    _check_state(lmmaes_tell(state, x, f), O.tell(s, x.numpy(), f.numpy()))


def test_recovery():
    torch.manual_seed(1)
    d = 80
    state = lmmaes(center_init=torch.zeros(d, dtype=F64), stdev_init=1.0, objective_sense="min", popsize=8, num_vectors=5)
    for _ in range(9):  # M filled past k = m
        x = lmmaes_ask(state)
        state = lmmaes_tell(state, x, (x**2 * torch.arange(1, d + 1)).sum(-1))
    z = torch.randn(1, state.popsize, d, dtype=F64)
    x = L._ask_torch(state, z)
    zr = L._recovered_steps(state, x)
    assert (x[0] - torch.as_tensor(O.ask(_oracle_state(state), z[0].numpy()))).abs().max() <= 1e-12 * x.abs().max()
    assert (zr - z).abs().max() <= 1e-13 * z.abs().max()
    np.testing.assert_allclose(O.recover(_oracle_state(state), O.steps(_oracle_state(state), z[0].numpy())), z[0].numpy(), rtol=0, atol=1e-13)


def test_item_independence():
    torch.manual_seed(2)
    B, d = 4, 48
    centers = torch.randn(B, d, dtype=F64)
    sigmas = torch.tensor([0.5, 1.0, 2.0, 0.1], dtype=F64)
    batched = lmmaes(center_init=centers, stdev_init=sigmas, objective_sense="min", popsize=8, num_vectors=4)
    singles = [lmmaes(center_init=centers[b], stdev_init=sigmas[b], objective_sense="min", popsize=8, num_vectors=4) for b in range(B)]
    for _ in range(7):
        x = lmmaes_ask(batched)
        f = (x**2).sum(-1) + torch.arange(B, dtype=F64)[:, None] * x[..., 0]
        batched = lmmaes_tell(batched, x, f)
        for b in range(B):
            singles[b] = lmmaes_tell(singles[b], x[b], f[b])
            for name in ("center", "sigma", "p_sigma", "M", "G"):
                a, e = getattr(batched, name)[b], getattr(singles[b], name)
                assert torch.allclose(a, e, rtol=1e-14, atol=1e-15), name


def test_batch_shape_broadcast():
    s = lmmaes(center_init=torch.zeros(3, 1, 40, dtype=F64), stdev_init=torch.ones(3, 2, dtype=F64), objective_sense="min")
    assert s.center.shape == (3, 2, 40) and s.M.shape == (3, 2, s.num_vectors, 40) and s.G.shape == (3, 2, s.num_vectors, s.num_vectors)
    x = lmmaes_ask(s)
    assert x.shape == (3, 2, s.popsize, 40)
    s2 = lmmaes_tell(s, x, x.sum(-1))
    assert s2.generation == 1 and s.generation == 0 and torch.all(s.M == 0)


def test_abi_return_codes():
    from evotorch_b200 import _native as nat

    if not nat.available():
        pytest.skip("libevok.so is not built")
    lib = nat.lib()
    consts = (nat.ctypes.c_double * 10)(*([0.1] * 10))
    p = 256  # any non-null address: argument checks come before any use
    ask = lambda *a: lib.evok_lmmaes_ask_batched(*a)  # noqa: E731
    # X, y, sigma, M, G, n_items, n_rows, D, m, k, consts, seed, stream_id0, ws, ws_bytes, stream
    assert ask(None, p, p, p, p, 1, 8, 40, 4, 0, consts, 0, 0, p, 1 << 20, None) == -1
    assert ask(p, p, p, p, p, 1, 8, 40, 4, 0, None, 0, 0, p, 1 << 20, None) == -1
    assert ask(p, p, p, p, p, -1, 8, 40, 4, 0, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 1, 40, 4, 0, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 129, 400, 4, 0, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 8, 0, 4, 0, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 8, 40, 0, 0, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 8, 40, 65, 0, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 8, 40, 4, 5, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 8, 40, 4, -1, consts, 0, 0, p, 1 << 20, None) == -2
    assert ask(p, p, p, p, p, 1, 8, 40, 4, 2, consts, 0, 0, p, 16, None) == -4
    assert ask(p, p, p, p, p, 0, 8, 40, 4, 2, consts, 0, 0, p, 16, None) == 0
    tell = lambda *a: lib.evok_lmmaes_tell_batched(*a)  # noqa: E731
    # X, aw, y, sigma, p_sigma, M, G, n_items, n_rows, D, m, k, consts, y', sigma', p_sigma', M', G', ws, ws_bytes, stream
    ok = (p, p, p, p, p, p, p, 1, 8, 40, 4, 2, consts, p, p, p, p, p, p, 1 << 20, None)
    for i in (0, 1, 2, 3, 4, 5, 6, 12, 13, 14, 15, 16, 17, 18):
        args = list(ok)
        args[i] = None
        assert tell(*args) == -1, i
    for i, v in ((7, -1), (8, 1), (8, 129), (9, 0), (10, 0), (10, 65), (11, 5), (11, -1)):
        args = list(ok)
        args[i] = v
        assert tell(*args) == -2, (i, v)
    args = list(ok)
    args[19] = 16
    assert tell(*args) == -4
    assert lib.evok_lmmaes_workspace_bytes(2, 8, 1000, 4) >= 2 * 4 * (2 * 4 * 8 + 1000)
