"""Separable CMA-ES on the fused path (`CMAES(..., separable=True)` on CUDA float32): the three kernels (`sample_eval_sq`,
`sepcma_moments`, `sepcma_update`), the searcher against the op-by-op mirror of the reference and a float64 restatement of the
reference's separable branch (cmaes.py:408-606, `_limit_stdev` cmaes.py:49-79), the lazy population, CUDA-graph replay and
checkpoint / resume.

The float64 restatement lives here, beside its only users; it is checked against the reference's own CPU run
(tests/golden/cmaes_variants_golden.npz, "separable/*") by the first test.
"""

import math
import os
import pickle

import numpy as np
import pytest
import torch

from evotorch_b200 import Problem, ops
from evotorch_b200.algorithms import CMAES
from oracle import es_oracle as O

DEV = "cuda"


def C(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def close(a, b, rtol=1e-5, atol=1e-6):
    np.testing.assert_allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=rtol, atol=atol)


# ------------------------------------------------------------------------------------------------ float64 restatement
class SepCMA64:
    """State and hyper-parameters of the reference's CMAES with separable=True (cmaes.py:279-385), state in float64.  The
    weights are formed in float32 like the reference's (make_tensor of float64 values into the problem dtype)."""

    def __init__(self, d, popsize, stdev_init, center, *, active=True, c_m=1.0, csa_squared=False, stdev_min=None, stdev_max=None,
                 limit_C_decomposition=True):
        f32 = np.float32
        self.d, self.popsize, self.mu_count = int(d), int(popsize), int(math.floor(popsize / 2))
        raw = (np.log((popsize + 1) / 2) - np.log(np.arange(popsize, dtype=np.float64) + 1)).astype(f32)
        pos, neg = raw[: self.mu_count], raw[self.mu_count:]
        mu_eff = float(np.sum(pos, dtype=f32) ** 2 / np.sum(pos**2, dtype=f32))
        self.c_m, self.active, self.csa_squared = c_m, active, csa_squared
        self.stdev_min, self.stdev_max = stdev_min, stdev_max
        self.c_sigma = (mu_eff + 2.0) / (d + mu_eff + 3)
        self.damp_sigma = 1 + 2 * max(0.0, math.sqrt((mu_eff - 1) / (d + 1)) - 1) + self.c_sigma
        self.c_c = (1 + (1 / d) + (mu_eff / d)) / (d**0.5 + (1 / d) + 2 * (mu_eff / d))
        self.c_1 = 1.0 / (d + 2.0 * np.sqrt(d) + mu_eff / d)
        self.c_mu = (0.25 + mu_eff + (1.0 / mu_eff) - 2) / (d + 4 * np.sqrt(d) + (mu_eff / 2.0))
        self.vd_sigma = math.sqrt(self.c_sigma * (2 - self.c_sigma) * mu_eff)
        self.vd_c = math.sqrt(self.c_c * (2 - self.c_c) * mu_eff)
        pos = pos / np.sum(pos, dtype=f32)
        if active:
            mu_eff_neg = float(np.sum(neg, dtype=f32) ** 2 / np.sum(neg**2, dtype=f32))
            alpha = min(1 + self.c_1 / self.c_mu, 1 + 2 * mu_eff_neg / (mu_eff + 2), (1 - self.c_mu - self.c_1) / (d * self.c_mu))
            neg = f32(alpha) * neg / np.sum(np.abs(neg), dtype=f32)
        else:
            neg = np.zeros_like(neg)
        self.weights = np.concatenate([pos, neg]).astype(f32).astype(np.float64)
        self.unbiased_expectation = math.sqrt(d) * (1 - (1 / (4 * d)) + 1 / (21 * d**2))
        if limit_C_decomposition:
            b = 10 * d * (self.c_1 + self.c_mu)
            b = b if abs(b) >= 1e-8 else (1e-8 if b >= 0 else -1e-8)
            self.decompose_C_freq = max(1, int(math.floor(1 / b)))
        else:
            self.decompose_C_freq = 1
        self.m = np.asarray(center, np.float64).copy()
        self.sigma = float(stdev_init)
        self.C, self.A = np.ones(d), np.ones(d)
        self.p_sigma, self.p_c = np.zeros(d), np.zeros(d)
        self.steps = 0

    def assign_weights(self, f, sense):
        """get_population_weights (cmaes.py:432-452): stable best-first order, weight of a solution = weights[its rank]."""
        order = O.argsort_for_ranking(np.asarray(f, np.float32), higher_is_better=(sense == "min"))
        ranks = np.empty(len(f), dtype=np.int64)
        ranks[order] = np.arange(len(f))
        return self.weights[ranks]

    def moments(self, Z, aw):
        """sum a_i z_i, sum b_i z_i^2, sum b_i (a = positive part, b = active-reweighted weights, cmaes.py:468-475, :531-535)."""
        Z = np.asarray(Z, np.float64)
        a = np.maximum(aw, 0.0)
        b = np.where(aw > 0, aw, self.d * aw / (Z * Z).sum(axis=1)) if self.active else aw
        return a @ Z, b @ (Z * Z), float(b.sum())

    def update(self, local, S2, wsum):
        """cmaes.py:454-565, separable branch, after the moments; shaped = A * local, sum_i b_i y_i^2 = A^2 * S2."""
        d = self.d
        shaped = self.A * local
        self.m = self.m + self.c_m * self.sigma * shaped
        self.p_sigma = (1 - self.c_sigma) * self.p_sigma + self.vd_sigma * local
        pnorm = float(np.linalg.norm(self.p_sigma))
        expo = (pnorm**2 / d - 1) / 2 if self.csa_squared else pnorm / self.unbiased_expectation - 1
        self.sigma = self.sigma * math.exp((self.c_sigma / self.damp_sigma) * expo)
        squared_sum = pnorm**2 / (1 - (1 - self.c_sigma) ** (2 * self.steps + 1))
        h_sig = 1.0 if (squared_sum / d) - 1 < 1 + 4.0 / (d + 1) else 0.0
        self.p_c = (1 - self.c_c) * self.p_c + h_sig * self.vd_c * shaped
        c1a = self.c_1 * (1 - (1 - h_sig**2) * self.c_c * (2 - self.c_c))
        # the separable branch: no weighted_pc factor in r1, and rmu subtracts the sum of the ACTIVE-reweighted weights
        self.C = self.C + c1a * (self.p_c**2 - self.C) + self.c_mu * (self.A**2 * S2 - wsum * self.C)
        if self.stdev_min is not None or self.stdev_max is not None:
            stdevs = np.clip(self.sigma * np.sqrt(self.C), self.stdev_min, self.stdev_max)
            self.C = (stdevs / self.sigma) ** 2
        if (self.steps + 1) % self.decompose_C_freq == 0:
            self.A = np.sqrt(self.C)
        self.steps += 1

    def step(self, Z, f, sense):
        self.update(*self.moments(Z, self.assign_weights(f, sense)))


def _torch_sphere(x):
    return torch.sum(x**2, dim=-1)


# ------------------------------------------------------------------------------------------------ CPU
def test_separable_oracle_reproduces_the_reference_run():
    """The float64 restatement fed with the z draws of the CPU op-by-op run and its fitnesses reproduces the reference's own
    separable run (same seed -> same torch-generator stream) for all 7 generations."""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "cmaes_variants_golden.npz"))
    prob = Problem("min", _torch_sphere, initial_bounds=(-3, 3), solution_length=8, vectorized=True, seed=11, dtype=torch.float32)
    c = CMAES(prob, stdev_init=1.0, popsize=14, separable=True)
    drawn = []
    sample = c.sample_distribution

    def recording(num_samples=None):
        zs, ys, xs = sample(num_samples)
        drawn.append(zs.clone())
        return zs, ys, xs

    c.sample_distribution = recording
    st = SepCMA64(8, 14, 1.0, c.m.numpy())
    close(st.weights, c.weights.numpy(), rtol=2e-6, atol=1e-8)
    assert st.decompose_C_freq == c.decompose_C_freq
    for t in range(7):
        c.step()
        st.step(drawn[-1].numpy(), c.population.evals[:, 0].numpy(), "min")
        close(c.population.evals[:, 0].numpy(), gold["separable/f"][t], rtol=2e-5, atol=2e-5)
        close(st.m, gold["separable/m"][t], rtol=2e-5, atol=5e-6)
        close(st.sigma, float(gold["separable/sigma"][t]), rtol=2e-5)
        close(st.C, gold["separable/C"][t], rtol=5e-5, atol=5e-6)
        close(st.p_sigma, gold["separable/p_sigma"][t], rtol=5e-5, atol=5e-6)
        close(st.p_c, gold["separable/p_c"][t], rtol=5e-5, atol=5e-6)


def test_lazy_separable_population_needs_the_fused_prerequisites():
    """A lazy population has no stand-in: building a separable searcher on one that the fused sampler cannot draw (CPU, a
    custom objective) fails loudly.  A non-separable searcher keeps a materialised population, as before."""
    from evotorch_b200.objectives import rastrigin

    cpu = Problem("min", rastrigin, initial_bounds=(-1, 1), solution_length=8, lazy_population=True, seed=1)
    with pytest.raises(ValueError, match="lazy population"):
        CMAES(cpu, stdev_init=1.0, popsize=10, separable=True)
    custom = Problem("min", _torch_sphere, initial_bounds=(-1, 1), solution_length=8, vectorized=True, lazy_population=True, seed=1)
    with pytest.raises(ValueError, match="lazy population"):
        CMAES(custom, stdev_init=1.0, popsize=10, separable=True)
    full = CMAES(cpu, stdev_init=1.0, popsize=10)
    full.step()
    assert full.population.values.shape == (10, 8)


def test_getstate_drops_the_fused_buffers_and_the_graph():
    """Pickles hold the search state, not the fused generation's scratch buffers or graph: those (and s = sigma * A) are
    rebuilt on the first step after loading.  The device-side step counter of a captured generation belongs to its graph,
    not to these buffers."""
    prob = Problem("min", _torch_sphere, initial_bounds=(-3, 3), solution_length=6, vectorized=True, seed=2, dtype=torch.float32)
    c = CMAES(prob, stdev_init=0.8, popsize=10, separable=True)
    c.step()
    fs = c._fused_state()  # the buffers exist whether or not this device runs the fused path
    assert set(fs) >= {"q", "aw", "local", "S2", "wsum", "s"}
    assert torch.equal(fs["s"], c.sigma * c.A)
    state = c.__getstate__()
    assert state["_fused"] is None and state["_graph"] is None and "_graph_workspaces" not in state
    for key in ("m", "sigma", "C", "A", "p_sigma", "p_c", "_population", "_problem"):
        assert key in state
    c._fused = None
    clone = pickle.loads(pickle.dumps(c))
    assert clone._fused is None
    clone.step(); c.step()
    assert torch.equal(clone.m, c.m) and torch.equal(clone.C, c.C) and float(clone.sigma) == float(c.sigma)


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _z(n, D, seed, stream_id, row0=0, offset=None):
    """The sampler's own normals (mu = 0, sigma = 1: fmaf(1, z, 0) == z)."""
    Z = torch.empty(n, D, device=DEV)
    ops.sample_eval(ops.OBJ_NONE, Z, torch.zeros(D, device=DEV), torch.ones(D, device=DEV), n_rows=n, symmetric=False, seed=seed,
                    stream_id=stream_id, row0=row0, stream_offset=offset)
    return Z


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(384, 96), (257, 1001), (1000, 4096)])
@pytest.mark.parametrize("row0,off", [(0, None), (6, 3)])
def test_sample_eval_sq_is_the_sampler_plus_squared_norms(shape, row0, off):
    """X and f bit-identical to evok_sample_eval (D % 4 == 0 and ragged D, X = NULL, nonzero row0, a device stream offset);
    q = sum_j z_ij^2 against float64 sums of the sampler's own z and of the oracle's Philox normals."""
    n, D = shape
    g = torch.Generator(device=DEV).manual_seed(n + D)
    mu = torch.randn(D, device=DEV, generator=g)
    sg = torch.rand(D, device=DEV, generator=g) + 0.3
    offset = None if off is None else torch.tensor([off], dtype=torch.int32, device=DEV)
    kw = dict(n_rows=n, seed=1234, stream_id=7, row0=row0, stream_offset=offset)
    for obj in (ops.OBJ_NONE, ops.OBJ_SPHERE, ops.OBJ_RASTRIGIN, ops.OBJ_ACKLEY):
        X, X2 = torch.empty(n, D, device=DEV), torch.empty(n, D, device=DEV)
        f = None if obj == ops.OBJ_NONE else torch.empty(n, device=DEV)
        f2 = None if obj == ops.OBJ_NONE else torch.empty(n, device=DEV)
        q = torch.full((n,), float("nan"), device=DEV)
        ops.sample_eval(obj, X, mu, sg, symmetric=False, f=f, **kw)
        ops.sample_eval_sq(obj, X2, mu, sg, q, f=f2, **kw)
        assert torch.equal(X, X2)
        if f is not None:
            assert torch.equal(f, f2)
            q2, f3 = torch.empty_like(q), torch.empty_like(f)
            ops.sample_eval_sq(obj, None, mu, sg, q2, f=f3, **kw)  # lazy: nothing written but f and q
            assert torch.equal(f, f3) and torch.equal(q, q2)
    Z = _z(n, D, 1234, 7, row0, offset).double()
    ref = (Z * Z).sum(dim=1)
    assert float(((q.double() - ref).abs() / ref).max()) < 1e-6
    rows = np.arange(0, n, max(1, n // 64))
    Zo = O.philox_normals(1234, 7 + (off or 0), row0 + rows, D)
    ref_o = (Zo * Zo).sum(axis=1)
    rel = np.abs(N(q)[rows].astype(np.float64) - ref_o) / ref_o
    assert float(rel.max()) < 1e-5, float(rel.max())


def _weights(n, active):
    st = SepCMA64(16, n, 1.0, np.zeros(16), active=active)
    return st.weights


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(384, 96), (1000, 1001), (20000, 2000)])
@pytest.mark.parametrize("active", [0, 1])
def test_sepcma_moments_match_float64(shape, active):
    """local = sum a_i z_i, S2 = sum b_i z_i^2, wsum = sum b_i with z regenerated from the sampler's counters, against float64
    sums over the sampler's own z, on both sides of the launch geometry; rows whose weight is zero are never regenerated: a NaN
    norm on them changes nothing."""
    n, D = shape
    g = torch.Generator(device="cpu").manual_seed(n)
    w = _weights(n, bool(active))
    aw = w[torch.randperm(n, generator=g).numpy()]
    aw[np.arange(n) % 17 == 5] = 0.0  # zero weights in both modes (with `active` the ones of the odd-size middle rank)
    offset = torch.tensor([2], dtype=torch.int32, device=DEV)
    q = torch.empty(n, device=DEV)
    mu, one = torch.zeros(D, device=DEV), torch.ones(D, device=DEV)
    ops.sample_eval_sq(ops.OBJ_NONE, torch.empty(n, D, device=DEV), mu, one, q, n_rows=n, seed=99, stream_id=5, row0=0, stream_offset=offset)
    awt = C(aw)
    local, S2, wsum = ops.sepcma_moments(awt, q, bool(active), D, seed=99, stream_id=5, stream_offset=offset)
    Z = _z(n, D, 99, 5, 0, offset).double()
    awd = awt.double()
    a = awd.clamp_min(0.0)
    b = torch.where(awd > 0, awd, D * awd / q.double()) if active else awd
    ref_l, ref_s2 = a @ Z, b @ (Z * Z)
    scale_l, scale_s2 = a.abs() @ Z.abs(), b.abs() @ (Z * Z)
    assert bool(((local.double() - ref_l).abs() <= 2e-5 * scale_l + 1e-12).all())
    assert bool(((S2.double() - ref_s2).abs() <= 2e-5 * scale_s2 + 1e-12).all())
    close(float(wsum), float(b.sum()), rtol=1e-5, atol=1e-6 * float(b.abs().sum()))
    q_nan = q.clone()
    q_nan[awt == 0] = float("nan")
    l2, s2b, w2 = ops.sepcma_moments(awt, q_nan, bool(active), D, seed=99, stream_id=5, stream_offset=offset)
    assert torch.equal(l2, local) and torch.equal(s2b, S2) and torch.equal(w2, wsum)


def _consts(st):
    return (st.c_m, st.c_sigma, st.damp_sigma, st.c_c, st.c_1, st.c_mu, st.vd_sigma, st.vd_c, st.unbiased_expectation, float(st.weights.sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [{}, {"stdev_min": 0.55, "stdev_max": 0.8}, {"csa_squared": True}, {"freq": 3, "steps": 4}, {"freq": 3, "steps": 5}])
def test_sepcma_update_matches_the_float64_step(kw):
    """evok_sepcma_update (one CTA) against the float64 restatement of the separable update, from a non-trivial state: with and
    without stdev bounds, squared CSA, a decomposition frequency > 1 on a generation that skips (steps 4) and one that takes
    (steps 5) the square root; the step count comes from the device counter, which the kernel advances."""
    kw = dict(kw)
    freq, steps = kw.pop("freq", 1), kw.pop("steps", 2)
    D, n = 1001, 600
    rng = np.random.default_rng(D + steps)
    st = SepCMA64(D, n, 0.7, rng.uniform(-1, 1, D), **kw)
    st.decompose_C_freq, st.steps = freq, steps
    st.C = rng.uniform(0.5, 1.5, D)
    st.A = np.sqrt(rng.uniform(0.5, 1.5, D))  # A need not be sqrt(C) between decompositions
    st.p_sigma, st.p_c = rng.standard_normal(D) * 0.3, rng.standard_normal(D) * 0.1
    f32 = lambda x: np.asarray(x, np.float32)  # noqa: E731
    for name in ("m", "C", "A", "p_sigma", "p_c"):
        setattr(st, name, f32(getattr(st, name)).astype(np.float64))
    st.sigma = float(np.float32(st.sigma))
    local, S2, wsum = f32(rng.standard_normal(D) * 0.4), f32(rng.uniform(0.2, 2.0, D)), f32([0.37])
    m, p_sigma, p_c, Cd, A = (C(getattr(st, k)) for k in ("m", "p_sigma", "p_c", "C", "A"))
    sigma = C([st.sigma])
    s = sigma * A
    m_prev, s_prev = torch.empty_like(m), torch.empty_like(m)
    m0, s0 = m.clone(), s.clone()
    steps_dev = torch.tensor([steps], dtype=torch.int64, device=DEV)
    ops.sepcma_update(C(local), C(S2), C(wsum), m, p_sigma, p_c, sigma, Cd, A, s, _consts(st), st.csa_squared, decompose_C_freq=freq,
                      steps=0, steps_dev=steps_dev, stdev_min=st.stdev_min, stdev_max=st.stdev_max, m_prev=m_prev, s_prev=s_prev)
    A_before = st.A.copy()
    st.update(local.astype(np.float64), S2.astype(np.float64), float(wsum[0]))
    assert int(steps_dev) == steps + 1
    assert torch.equal(m_prev, m0) and torch.equal(s_prev, s0)
    close(N(m), st.m, rtol=2e-5, atol=2e-6)
    close(float(sigma), st.sigma, rtol=2e-5)
    close(N(p_sigma), st.p_sigma, rtol=2e-5, atol=2e-6)
    close(N(p_c), st.p_c, rtol=2e-5, atol=2e-6)
    close(N(Cd), st.C, rtol=2e-5, atol=2e-6)
    close(N(A), st.A, rtol=2e-5, atol=2e-6)
    assert torch.equal(s, sigma * A)
    if freq > 1 and (steps + 1) % freq != 0:
        assert np.array_equal(N(A), A_before.astype(np.float32))


# ------------------------------------------------------------------------------------------------ GPU: searcher
def _sep(seed=5, D=96, n=384, fused=True, graph=False, lazy=False, obj="sphere", **kw):
    from evotorch_b200 import objectives

    prob = Problem("min", getattr(objectives, obj), initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=seed, lazy_population=lazy)
    c = CMAES(prob, stdev_init=1.0, popsize=n, separable=True, **kw)
    if not fused:
        c._fused_ok = lambda: False  # the op-by-op mirror of the reference's _step
    if graph:
        c.enable_cuda_graph()
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [{}, {"active": False}, {"csa_squared": True}, {"limit_C_decomposition": False},
                                {"stdev_min": 0.9, "stdev_max": 1.05}])
def test_separable_fused_generation_equals_the_op_by_op_path(kw):
    """Same seed, same Philox stream id per generation (so the same z): the fused separable generation against the op-by-op
    mirror of the reference's _step over 6 generations."""
    a, b = _sep(fused=True, **kw), _sep(fused=False, **kw)
    for _ in range(6):
        a.step(); b.step()
        assert a._fused is not None and b._fused is None
        close(N(a.m), N(b.m), rtol=2e-5, atol=2e-6)
        close(float(a.sigma), float(b.sigma), rtol=2e-5)
        close(N(a.p_sigma), N(b.p_sigma), rtol=2e-5, atol=2e-5)
        close(N(a.p_c), N(b.p_c), rtol=2e-5, atol=2e-5)
        close(N(a.C), N(b.C), rtol=2e-5, atol=2e-6)
        close(N(a.A), N(b.A), rtol=2e-5, atol=2e-6)
    assert a._problem._philox_stream == b._problem._philox_stream == 6


@pytest.mark.gpu
def test_separable_generation_at_4096_x_2000_matches_the_float64_oracle():
    """One fused generation from a non-trivial diagonal covariance against the float64 restatement, fed with the z of the same
    Philox stream (the sampler's own normals) and the fused evaluation's fitnesses: m, sigma, C, A within 2e-5."""
    D, n = 2000, 4096
    rng = np.random.default_rng(11)
    c = _sep(seed=3, D=D, n=n)
    C0 = rng.uniform(0.3, 2.0, D).astype(np.float32)
    c.C, c.A = C(C0), torch.sqrt(C(C0))
    st = SepCMA64(D, n, 1.0, N(c.m))
    st.C, st.A = C0.astype(np.float64), N(c.A).astype(np.float64)
    prob = c._problem
    seed, sid = prob._philox_seed, prob._philox_stream
    c.step()
    Z = N(_z(n, D, seed, sid)).astype(np.float64)
    st.step(Z, N(c.population.evals[:, 0]), "min")
    close(N(c.m), st.m, rtol=2e-5, atol=2e-6)
    close(float(c.sigma), st.sigma, rtol=2e-5)
    close(N(c.C), st.C, rtol=2e-5, atol=2e-6)
    close(N(c.A), st.A, rtol=2e-5, atol=2e-6)


_STATE = ("m", "sigma", "C", "A", "p_sigma", "p_c")


def _same_state(a, b):
    for k in _STATE:
        assert torch.equal(getattr(a, k), getattr(b, k)), k


@pytest.mark.gpu
def test_lazy_population_equals_the_materialised_one_bit_for_bit():
    """Same z, same f, same sums: the lazy run is the materialised run, and its population regenerates the rows that were actually
    evaluated (drawn from the centre / stdev before the update), so `values` and `pop_best` agree after every step.  The centre is
    given: a materialised searcher draws its initial population from the torch generator before a random centre, a lazy one
    does not."""
    m0 = C(np.random.default_rng(4).uniform(-3, 3, 301))
    mat, lazy = _sep(D=301, n=1000, obj="rastrigin", center_init=m0), _sep(D=301, n=1000, obj="rastrigin", lazy=True, center_init=m0)
    from evotorch_b200.core import LazySolutionBatch

    assert isinstance(lazy.population, LazySolutionBatch) and not isinstance(mat.population, LazySolutionBatch)
    for _ in range(8):
        mat.step(); lazy.step()
        _same_state(mat, lazy)
        assert torch.equal(mat.population.evals, lazy.population.evals)
        assert torch.equal(mat.population.values, lazy.population.values)
        assert torch.equal(mat.status["pop_best"].values, lazy.status["pop_best"].values)
        assert mat.status["pop_best_eval"] == lazy.status["pop_best_eval"]
        close(O.rastrigin(N(lazy.population.values)), N(lazy.population.evals[:, 0]), rtol=1e-5, atol=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["plain", "freq3_bounds", "lazy"])
def test_separable_graph_replay_equals_eager_fused_stepping(case):
    """`enable_cuda_graph()` on separable runs, bit for bit against eager fused stepping over 8 generations: any decomposition
    frequency (the device step counter drives it), stdev bounds, and a lazy population whose `values` follow the replays."""
    kw = dict(D=200, n=600)
    if case == "freq3_bounds":
        kw.update(stdev_min=0.9, stdev_max=1.02)
    lazy = case == "lazy"
    a, b = _sep(lazy=lazy, **kw), _sep(lazy=lazy, graph=True, **kw)
    if case == "freq3_bounds":
        a.decompose_C_freq = b.decompose_C_freq = 3
    for g in range(8):
        a.step(); b.step()
        _same_state(a, b)
        assert torch.equal(a.population.evals, b.population.evals), g
        if lazy:
            assert torch.equal(a.population.values, b.population.values), g
    assert b._graph is not None and b.status["iter"] == 8
    assert a._problem._philox_stream == b._problem._philox_stream


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eager", "lazy_graph"])
def test_separable_checkpoint_resume_is_bit_identical(mode, tmp_path):
    """PicklingLogger(checkpoint=True) mid-run: the resumed searcher rebuilds its buffers and s = sigma * A and continues exactly
    like the uninterrupted run."""
    from evotorch_b200.logging import PicklingLogger

    def make():
        return _sep(D=150, n=500, obj="rastrigin", lazy=mode.startswith("lazy"), graph=mode.endswith("graph"))

    straight = make()
    straight.run(11)
    s = make()
    logger = PicklingLogger(s, interval=5, directory=str(tmp_path), prefix="sep", verbose=False, checkpoint=True)
    s.run(5)
    resumed = PicklingLogger.resume(logger.last_file_name)
    assert resumed._graph is None and resumed._fused is None and resumed.step_count == 5
    resumed.run(6)
    _same_state(resumed, straight)
    assert torch.equal(resumed.population.evals, straight.population.evals)


@pytest.mark.gpu
def test_lazy_separable_run_needs_no_population_memory():
    """262 144 x 4 096 (4 GB if materialised): a lazy separable run stays within 64 MB of the memory in use before the searcher
    was built."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    from evotorch_b200.objectives import rastrigin

    prob = Problem("min", rastrigin, initial_bounds=(-3, 3), solution_length=4096, device=DEV, seed=1, lazy_population=True)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    c = CMAES(prob, stdev_init=1.0, popsize=262_144, separable=True)
    for _ in range(3):
        c.step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 64 * 2**20, peak
    assert math.isfinite(float(c.sigma))
