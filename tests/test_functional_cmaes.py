"""Functional CMA-ES, generic torch path (CPU, float64): every item of a batched search against the float64 oracle of the
non-separable update, generation by generation from a common state; the constants against the CMAES class; argument errors."""

import numpy as np
import pytest
import torch

from evotorch_b200 import Problem
from evotorch_b200.algorithms import CMAES
from evotorch_b200.algorithms.functional import CMAESState, cmaes, cmaes_ask, cmaes_tell
from oracle import es_oracle as O

STATE = ("center", "sigma", "C", "A", "p_sigma", "p_c")


def ellipsoid(x):
    d = x.shape[-1]
    return ((10.0 ** (3 * torch.arange(d, dtype=x.dtype) / max(d - 1, 1))) * x * x).sum(-1)


def oracle_state(state: CMAESState, b: int) -> O.CMAESState:
    """The oracle holding item b of `state` (its fp32 arrays) with the state's own learning rates and weights."""
    hp = state.hyperparameters
    B, d = -1, state.center.shape[-1]
    item = {name: getattr(state, name).reshape((B,) + tuple(getattr(state, name).shape[state.center.ndim - 1:]))[b] for name in STATE}
    o = O.CMAESState(d, hp.popsize, float(item["sigma"]), item["center"].numpy(), active=state.active, csa_squared=state.csa_squared,
                     stdev_min=state.stdev_min, stdev_max=state.stdev_max)
    o.c_m, o.c_sigma, o.damp_sigma, o.c_c, o.c_1, o.c_mu = hp.c_m, hp.c_sigma, hp.damp_sigma, hp.c_c, hp.c_1, hp.c_mu
    o.variance_discount_sigma, o.variance_discount_c, o.unbiased_expectation = hp.variance_discount_sigma, hp.variance_discount_c, hp.unbiased_expectation
    o.weights, o.decompose_C_freq, o.steps = hp.weights.numpy().astype(np.float32), hp.decompose_C_freq, state.generation
    o.m = item["center"].numpy().astype(np.float32)
    o.sigma = np.float32(item["sigma"].item())
    for name in ("p_sigma", "p_c", "C", "A"):
        setattr(o, name, item[name].numpy().astype(np.float32))
    return o


CONFIGS = [
    dict(),
    dict(active=False),
    dict(csa_squared=True, objective_sense="max"),
    dict(stdev_min=0.02, stdev_max=0.6),
    dict(c_1_ratio=0.1, c_mu_ratio=0.1),  # decompose_C_freq = 2 at D = 6: A is refactorised every other generation
    dict(c_1_ratio=0.1, c_mu_ratio=0.1, limit_C_decomposition=False),
]


@pytest.mark.parametrize("batch", [(), (3,), (2, 3)])
@pytest.mark.parametrize("config", range(len(CONFIGS)))
def test_torch_path_against_the_oracle(batch, config):
    kw = dict(objective_sense="min")
    kw.update(CONFIGS[config])
    sign = -1.0 if kw["objective_sense"] == "max" else 1.0
    d = 6
    g = torch.Generator().manual_seed(len(batch) * 10 + config)
    center = torch.randn(batch + (d,), generator=g, dtype=torch.float64)
    stdev = 0.2 + torch.rand(batch, generator=g, dtype=torch.float64) if batch else 0.3
    torch.manual_seed(config)
    state = cmaes(center_init=center, stdev_init=stdev, **kw)
    if "c_1_ratio" in kw:
        assert state.hyperparameters.decompose_C_freq == (2 if kw.get("limit_C_decomposition", True) else 1)
    n = state.popsize
    B = int(np.prod(batch)) if batch else 1
    for gen in range(10):
        x = cmaes_ask(state)
        assert x.shape == batch + (n, d) and x.dtype == torch.float64
        f = sign * ellipsoid(x)
        new = cmaes_tell(state, x, f)
        assert new.generation == gen + 1 and torch.equal(state.center.reshape(-1), center.reshape(-1)) == (gen == 0)
        xs, fs = x.reshape(B, n, d), f.reshape(B, n)
        for b in range(B):
            o = oracle_state(state, b)
            y = (xs[b] - torch.as_tensor(o.m, dtype=torch.float64)) / float(o.sigma)
            z = torch.linalg.solve_triangular(torch.as_tensor(o.A, dtype=torch.float64).T, y, upper=True, left=False)
            O.cmaes_update(o, z.numpy(), y.numpy(), O.cmaes_assign_weights(o, fs[b].numpy(), kw["objective_sense"]))
            got = {name: getattr(new, name).reshape((B,) + tuple(getattr(new, name).shape[new.center.ndim - 1:]))[b] for name in STATE}
            for name, ref in (("center", o.m), ("sigma", o.sigma), ("p_sigma", o.p_sigma), ("p_c", o.p_c), ("C", o.C), ("A", o.A)):
                ref = torch.as_tensor(np.asarray(ref, dtype=np.float64))
                tol = 1e-4 if name == "A" else 2e-5
                assert torch.allclose(got[name], ref, rtol=tol, atol=tol * float(ref.abs().max())), (gen, b, name)
        state = new  # the oracle adopts our state each generation: ranks may swap at the last bit


def test_constants_equal_those_of_the_class():
    d = 9
    for kw in (dict(), dict(popsize=14, c_m=0.8, c_sigma_ratio=1.3, damp_sigma_ratio=0.7, c_c_ratio=1.1, c_1_ratio=0.5, c_mu_ratio=0.6),
               dict(active=False, limit_C_decomposition=False), dict(c_1_ratio=0.05, c_mu_ratio=0.05)):
        prob = Problem("min", lambda x: (x * x).sum(-1), solution_length=d, initial_bounds=(-1, 1), vectorized=True)
        obj = CMAES(prob, stdev_init=1.0, center_init=torch.zeros(d), **kw)
        hp = cmaes(center_init=torch.zeros(d), stdev_init=1.0, objective_sense="min", **kw).hyperparameters
        assert hp.popsize == obj.popsize and hp.mu == obj.mu
        assert torch.equal(hp.weights, obj.weights) and hp.weights_sum == obj._weights_sum
        for name in ("mu_eff", "c_m", "c_sigma", "damp_sigma", "c_c", "c_1", "c_mu", "variance_discount_sigma", "variance_discount_c",
                     "unbiased_expectation", "decompose_C_freq"):
            assert getattr(hp, name) == getattr(obj, name), name


def test_state_shapes_and_broadcast_stdev():
    s = cmaes(center_init=torch.zeros(4, dtype=torch.float64), stdev_init=torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64),
              objective_sense="min")
    assert s.center.shape == (3, 4) and s.sigma.shape == (3,) and s.C.shape == (3, 4, 4) and s.A.shape == (3, 4, 4)
    assert s.p_sigma.shape == (3, 4) and s.generation == 0 and s.weights.shape == (s.popsize,)
    assert torch.equal(s.sigma, torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64))


def test_tell_leaves_the_given_state_unchanged():
    s = cmaes(center_init=torch.randn(2, 5, dtype=torch.float64), stdev_init=1.0, objective_sense="min")
    before = [getattr(s, name).clone() for name in STATE]
    x = cmaes_ask(s)
    cmaes_tell(s, x, ellipsoid(x))
    assert all(torch.equal(a, getattr(s, name)) for a, name in zip(before, STATE))


def test_argument_errors():
    c = torch.zeros(3, 5)
    with pytest.raises(ValueError, match="separable"):
        cmaes(center_init=c, stdev_init=1.0, objective_sense="min", separable=True)
    with pytest.raises(ValueError, match="per-item"):
        cmaes(center_init=c, stdev_init=1.0, objective_sense="min", c_1_ratio=torch.ones(3))
    with pytest.raises(ValueError, match="objective_sense"):
        cmaes(center_init=c, stdev_init=1.0, objective_sense="minimize")
    with pytest.raises(ValueError, match="center_init"):
        cmaes(center_init=torch.tensor(1.0), stdev_init=1.0, objective_sense="min")
    with pytest.raises(RuntimeError):
        cmaes(center_init=c, stdev_init=torch.ones(2), objective_sense="min")  # batch shapes (3,) and (2,) do not broadcast
    s = cmaes(center_init=c, stdev_init=1.0, objective_sense="min")
    x = cmaes_ask(s)
    with pytest.raises(ValueError, match="values"):
        cmaes_tell(s, x[:, :-1], ellipsoid(x)[:, :-1])
    with pytest.raises(ValueError, match="evals"):
        cmaes_tell(s, x, ellipsoid(x)[:2])
