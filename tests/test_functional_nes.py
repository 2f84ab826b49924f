"""Functional XNES and SNES off the kernels: constants and validation, one-item float64 tells against the object-API
distributions, the reference golden trajectories, item independence, the "max" sense, injected values and the ABI return codes."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200.algorithms.functional import snes, snes_ask, snes_tell, xnes, xnes_ask, xnes_tell
from evotorch_b200.algorithms.functional import funcxnes as X
from evotorch_b200.distributions import ExpGaussian, ExpSeparableGaussian
from evotorch_b200.tools.ranking import rank
from oracle import functional_nes_oracle as O

F64 = torch.float64


@pytest.fixture(scope="module")
def golden():
    import os

    return np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden.npz"))


def _close(a, b, rtol=1e-12):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(np.abs(b).max(), 1e-300)
    assert np.abs(a - b).max() <= rtol * scale, (np.abs(a - b).max(), scale)


@pytest.mark.parametrize("d", [1, 2, 5, 16, 96, 1000])
def test_constants(d):
    s = xnes(center_init=torch.zeros(d, dtype=F64), stdev_init=1.0, objective_sense="min")
    assert s.popsize == 4 + int(math.floor(3 * math.log(d))) and s.center_learning_rate == 1.0
    assert s.stdev_learning_rate == pytest.approx(0.6 * (3 + math.log(d)) / (d * math.sqrt(d)), rel=1e-15)
    s2 = xnes(center_init=torch.zeros(d, dtype=F64), stdev_init=1.0, objective_sense="min", stdev_learning_rate=0.5)
    assert s2.stdev_learning_rate == pytest.approx(0.5 * s.stdev_learning_rate, rel=1e-15)
    s3 = xnes(center_init=torch.zeros(d, dtype=F64), stdev_init=1.0, objective_sense="min", stdev_learning_rate=0.5, scale_learning_rate=False)
    assert s3.stdev_learning_rate == 0.5
    n = snes(center_init=torch.zeros(d, dtype=F64), stdev_init=1.0, objective_sense="min")
    assert n.popsize == s.popsize and n.center_learning_rate == 1.0 and n.ranking_method == "nes"
    assert n.stdev_learning_rate == pytest.approx(0.2 * (3 + math.log(d)) / math.sqrt(d), rel=1e-15)


def test_initial_state_and_batch_shape():
    s = xnes(center_init=torch.zeros(3, 1, 4, dtype=F64), stdev_init=torch.tensor([[1.0, 2.0, 3.0, 4.0], [0.5, 0.5, 0.5, 0.5]], dtype=F64),
             objective_sense="min")
    assert s.center.shape == (3, 2, 4) and s.A.shape == (3, 2, 4, 4) and s.A_inv.shape == (3, 2, 4, 4)
    assert torch.equal(s.A[1, 0], torch.diag(torch.tensor([1.0, 2.0, 3.0, 4.0], dtype=F64)))
    assert torch.allclose(s.A[2, 1] @ s.A_inv[2, 1], torch.eye(4, dtype=F64), rtol=0, atol=1e-15)
    x = xnes_ask(s)
    assert x.shape == (3, 2, s.popsize, 4)
    s1 = xnes_tell(s, x, x.sum(-1))
    assert s1.center.shape == (3, 2, 4) and torch.all(s.center == 0)
    n = snes(center_init=torch.zeros(2, 6, dtype=F64), stdev_init=torch.ones(5, 1, 6, dtype=F64), objective_sense="min")
    assert n.center.shape == (5, 2, 6) and n.stdev.shape == (5, 2, 6)
    assert snes_ask(n).shape == (5, 2, n.popsize, 6)


def test_validation():
    x0 = torch.zeros(5, dtype=F64)
    for make in (xnes, snes):
        with pytest.raises(ValueError, match="objective_sense"):
            make(center_init=x0, stdev_init=1.0, objective_sense="minimize")
        with pytest.raises(ValueError, match="popsize"):
            make(center_init=x0, stdev_init=1.0, objective_sense="min", popsize=1)
        with pytest.raises(ValueError, match="ranking"):
            make(center_init=x0, stdev_init=1.0, objective_sense="min", ranking_method="best")
    s = xnes(center_init=x0, stdev_init=1.0, objective_sense="min")
    with pytest.raises(ValueError, match="A_inv"):
        xnes_tell(s._replace(A_inv=torch.eye(4, dtype=F64)), xnes_ask(s), torch.zeros(s.popsize, dtype=F64))
    with pytest.raises(ValueError, match="`A`"):
        xnes_ask(s._replace(A=torch.eye(5, dtype=F64).expand(2, 5, 5)))
    x = xnes_ask(s)
    with pytest.raises(ValueError, match="values"):
        xnes_tell(s, x[:-1], torch.zeros(s.popsize - 1, dtype=F64))
    with pytest.raises(ValueError, match="evals"):
        xnes_tell(s, x, torch.zeros(s.popsize + 1, dtype=F64))
    n = snes(center_init=x0, stdev_init=1.0, objective_sense="min")
    with pytest.raises(ValueError, match="lazy=True"):
        from evotorch_b200.algorithms.functional import snes_ask_and_evaluate

        snes_ask_and_evaluate(n, objective=lambda v: v.sum(-1), lazy=True)


def test_restarts_rejects_nes_states():
    from evotorch_b200.algorithms.functional import restarts

    for make in (xnes, snes):
        with pytest.raises(TypeError, match="CMAESState or a SepCMAESState"):
            restarts(make(center_init=torch.zeros(40, dtype=F64), stdev_init=1.0, objective_sense="min"), lb=-1.0, ub=1.0)


@pytest.mark.parametrize("method", ["nes", "centered", "linear", "normalized", "raw"])
@pytest.mark.parametrize("maximize", [False, True])
def test_rank_rows(method, maximize):
    g = torch.Generator().manual_seed(7)
    f = torch.randn(5, 13, generator=g, dtype=F64)
    f[2, 3] = f[2, 7]  # a tie: ascending index order, as in the stable sort of tools.ranking
    w = X.rank_rows(f, method, maximize)
    for b in range(5):
        _close(w[b].numpy(), rank(f[b], method, higher_is_better=maximize).numpy(), rtol=1e-15)


def _random_xnes(d, popsize, seed, method="nes", maximize=False, B=1):
    g = torch.Generator().manual_seed(seed)
    s = xnes(center_init=torch.randn(B, d, generator=g, dtype=F64), stdev_init=1.0, objective_sense="max" if maximize else "min",
             popsize=popsize, ranking_method=method, stdev_learning_rate=0.3, scale_learning_rate=False, center_learning_rate=0.8)
    Q = torch.linalg.qr(torch.randn(B, d, d, generator=g, dtype=F64))[0]
    A = Q * torch.exp(torch.randn(B, 1, d, generator=g, dtype=F64))
    s = s._replace(A=A, A_inv=torch.linalg.inv(A))
    x = xnes_ask(s)
    f = (x**2).sum(-1) + x[..., 0]
    return s, x, f


@pytest.mark.parametrize("method", ["nes", "centered", "linear", "normalized"])
@pytest.mark.parametrize("maximize", [False, True])
def test_xnes_tell_equals_exp_gaussian(method, maximize):
    s, x, f = _random_xnes(7, 12, 3, method, maximize)
    s1 = xnes_tell(s, x, f)
    dist = ExpGaussian({"mu": s.center[0], "sigma": s.A[0], "sigma_inv": s.A_inv[0]}, dtype=F64)
    g = dist.compute_gradients(x[0], f[0], objective_sense="max" if maximize else "min", ranking_method=method)
    upd = dist.update_parameters(g, learning_rates={"mu": 0.8, "sigma": 0.3})
    _close(s1.center[0].numpy(), upd.mu.numpy())
    _close(s1.A[0].numpy(), upd.A.numpy())
    _close(s1.A_inv[0].numpy(), upd.A_inv.numpy())


@pytest.mark.parametrize("method", ["nes", "centered", "linear"])
@pytest.mark.parametrize("maximize", [False, True])
def test_snes_tell_equals_exp_separable(method, maximize):
    g = torch.Generator().manual_seed(4)
    d = 9
    s = snes(center_init=torch.randn(d, generator=g, dtype=F64), stdev_init=torch.rand(d, generator=g, dtype=F64) + 0.5, popsize=14,
             objective_sense="max" if maximize else "min", ranking_method=method, center_learning_rate=0.7, stdev_learning_rate=0.4,
             scale_learning_rate=False)
    x = snes_ask(s)
    f = (x**2).sum(-1)
    s1 = snes_tell(s, x, f)
    dist = ExpSeparableGaussian({"mu": s.center, "sigma": s.stdev}, dtype=F64)
    gr = dist.compute_gradients(x, f, objective_sense="max" if maximize else "min", ranking_method=method)
    upd = dist.update_parameters(gr, learning_rates={"mu": 0.7, "sigma": 0.4})
    _close(s1.center.numpy(), upd.mu.numpy())
    _close(s1.stdev.numpy(), upd.sigma.numpy())


def test_snes_stdev_bounds_against_oracle():
    g = torch.Generator().manual_seed(5)
    B, d = 3, 6
    s = snes(center_init=torch.randn(B, d, generator=g, dtype=F64), stdev_init=1.0, objective_sense="min", popsize=10, stdev_min=0.9,
             stdev_max=1.05, stdev_max_change=0.02)
    x = snes_ask(s)
    f = (x**2).sum(-1)
    s1 = snes_tell(s, x, f)
    mu, sig = O.snes_tell(s.center.numpy(), s.stdev.numpy(), x.numpy(), f.numpy(), maximize=False, ranking="nes", lr_mu=1.0,
                          lr_sigma=s.stdev_learning_rate, stdev_min=0.9, stdev_max=1.05, stdev_max_change=0.02)
    np.testing.assert_allclose(s1.center.numpy(), mu, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(s1.stdev.numpy(), sig, rtol=1e-5, atol=1e-6)
    assert np.all(s1.stdev.numpy() <= 1.02 + 1e-12) and np.all(s1.stdev.numpy() >= 0.98 - 1e-12)


def test_xnes_golden_trajectory(golden):
    mus, As, Xs, fs = (golden[f"traj/xnes/{k}"] for k in ("mu", "sigma", "X", "f"))
    s = xnes(center_init=torch.tensor(mus[0], dtype=F64), stdev_init=1.5, objective_sense="min", popsize=16)
    assert np.allclose(s.A.numpy(), As[0])
    for t in range(len(mus) - 1):
        s = xnes_tell(s, torch.tensor(Xs[t], dtype=F64), torch.tensor(fs[t], dtype=F64))
        np.testing.assert_allclose(s.center.numpy(), mus[t + 1], rtol=2e-4, atol=2e-5)
        np.testing.assert_allclose(s.A.numpy(), As[t + 1], rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("tag", ["snes", "snes_clipup"])
def test_snes_golden_trajectory(golden, tag):
    mus, sigs, Xs, fs = (golden[f"traj/{tag}/{k}"] for k in ("mu", "sigma", "X", "f"))
    kw = dict(optimizer="clipup", center_learning_rate=0.2, stdev_max_change=0.3) if tag == "snes_clipup" else {}
    s = snes(center_init=torch.tensor(mus[0], dtype=F64), stdev_init=torch.tensor(sigs[0], dtype=F64), objective_sense="min", popsize=24, **kw)
    for t in range(len(mus) - 1):
        s = snes_tell(s, torch.tensor(Xs[t], dtype=F64), torch.tensor(fs[t], dtype=F64))
        np.testing.assert_allclose(s.center.numpy(), mus[t + 1], rtol=2e-4, atol=2e-5)
        np.testing.assert_allclose(s.stdev.numpy(), sigs[t + 1], rtol=2e-4, atol=2e-5)


def test_xnes_against_oracle_batch():
    s, x, f = _random_xnes(6, 11, 8, B=4)
    s1 = xnes_tell(s, x, f)
    mu, A, A_inv = O.xnes_tell(s.center.numpy(), s.A.numpy(), s.A_inv.numpy(), x.numpy(), f.numpy(), maximize=False, ranking="nes", lr_mu=0.8,
                               lr_A=0.3)
    np.testing.assert_allclose(s1.center.numpy(), mu, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(s1.A.numpy(), A, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(s1.A_inv.numpy(), A_inv, rtol=1e-5, atol=1e-5)


def test_item_independence():
    B = 4
    s, _, _ = _random_xnes(5, 9, 11, B=B)
    singles = [s._replace(center=s.center[b], A=s.A[b], A_inv=s.A_inv[b]) for b in range(B)]
    n = snes(center_init=s.center, stdev_init=torch.tensor([0.5, 1.0, 2.0, 0.1], dtype=F64)[:, None] * torch.ones(5, dtype=F64),
             objective_sense="min", popsize=9)
    nsingles = [n._replace(center=n.center[b], stdev=n.stdev[b]) for b in range(B)]
    for _ in range(5):
        x = xnes_ask(s)
        f = (x**2).sum(-1) + torch.arange(B, dtype=F64)[:, None] * x[..., 0]
        s = xnes_tell(s, x, f)
        xs = snes_ask(n)
        fs = (xs**2).sum(-1) + torch.arange(B, dtype=F64)[:, None] * xs[..., 1]
        n = snes_tell(n, xs, fs)
        for b in range(B):
            singles[b] = xnes_tell(singles[b], x[b], f[b])
            nsingles[b] = snes_tell(nsingles[b], xs[b], fs[b])
            for name in ("center", "A", "A_inv"):
                assert torch.allclose(getattr(s, name)[b], getattr(singles[b], name), rtol=1e-13, atol=1e-15), name
            for name in ("center", "stdev"):
                assert torch.allclose(getattr(n, name)[b], getattr(nsingles[b], name), rtol=1e-13, atol=1e-15), name


def test_maximize_mirrors_minimize():
    s, x, f = _random_xnes(5, 10, 12)
    lo, hi = xnes_tell(s, x, f), xnes_tell(s._replace(maximize=True), x, -f)
    for name in ("center", "A", "A_inv"):
        assert torch.equal(getattr(lo, name), getattr(hi, name))


def test_injected_values():
    # the tell recovers z from the values, so a replaced row is told as what it is
    s, x, f = _random_xnes(6, 10, 13)
    x = x.clone()
    x[0, 0] = torch.linspace(-1, 1, 6, dtype=F64)
    x[0, 1] = torch.clamp(x[0, 1], -0.2, 0.2)
    f = (x**2).sum(-1)
    s1 = xnes_tell(s, x, f)
    dist = ExpGaussian({"mu": s.center[0], "sigma": s.A[0], "sigma_inv": s.A_inv[0]}, dtype=F64)
    upd = dist.update_parameters(dist.compute_gradients(x[0], f[0], objective_sense="min", ranking_method="nes"),
                                 learning_rates={"mu": 0.8, "sigma": 0.3})
    _close(s1.A[0].numpy(), upd.A.numpy())
    _close(s1.center[0].numpy(), upd.mu.numpy())


def test_xnes_solves_sphere_in_float64():
    torch.manual_seed(0)
    s = xnes(center_init=torch.full((3, 8), 3.0, dtype=F64), stdev_init=1.0, objective_sense="min")
    for _ in range(300):
        x = xnes_ask(s)
        s = xnes_tell(s, x, (x**2).sum(-1))
    assert torch.all((s.center**2).sum(-1) < 1e-4)


def test_abi_return_codes():
    from evotorch_b200 import _native as nat

    if not nat.available():
        pytest.skip("libevok.so is not built")
    lib = nat.lib()
    p = 256  # any non-null address: argument checks come before any use
    expm = lambda *a: lib.evok_sym_expm_pair_batched(*a)  # noqa: E731
    # S, n_items, D, F+, F-, stream
    for i in (0, 3, 4):
        args = [p, 1, 8, p, p, None]
        args[i] = None
        assert expm(*args) == -1, i
    for n_items, d in ((-1, 8), (1, 0), (1, 97)):
        assert expm(p, n_items, d, p, p, None) == -2
    assert expm(p, 0, 8, p, p, None) == 0
    tell = lambda *a: lib.evok_xnes_tell_batched(*a)  # noqa: E731
    # X, w, mu, A, A_inv, n_items, n_rows, D, lr_mu, lr_A, mu', A', A_inv', stream
    ok = (p, p, p, p, p, 1, 8, 16, 1.0, 0.1, p, p, p, None)
    for i in (0, 1, 2, 3, 4, 10, 11, 12):
        args = list(ok)
        args[i] = None
        assert tell(*args) == -1, i
    for i, v in ((5, -1), (6, 1), (7, 0), (7, 97)):
        args = list(ok)
        args[i] = v
        assert tell(*args) == -2, (i, v)
    args = list(ok)
    args[5] = 0
    assert tell(*args) == 0
