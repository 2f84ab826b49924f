"""Functional separable CMA-ES on the kernels: the batched moments against float64 (stored and rebuilt rows bit for bit, every
item the bits of a one-item call), item chunks past the grid limit, the batched update against the single call, sample-and-evaluate
against the ask, lazy runs against stored runs bit for bit, whole generations against the float64 reference per item, launch
counts that do not grow with the batch, no host synchronisation, and the memory of a lazy run."""

import math

import pytest
import torch

from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import LazyPopulation, sepcmaes, sepcmaes_ask, sepcmaes_ask_and_evaluate, sepcmaes_tell
from evotorch_b200.algorithms.functional.funccmaes import _consts
from evotorch_b200.objectives import FusedObjective, rastrigin
from oracle import functional_sepcma_oracle as SO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
EPS = 2.0 ** -24
SHIFTED_SPHERE = ({"s": "(x - o)**2"}, "s")


def gam(k):
    return k * EPS / (1 - k * EPS)


def _population(B, n, D, seed, sigma_scale=1.0):
    """(X stored by the batched sampler, m, s, seed): items with different centres and per-column stdevs."""
    g = torch.Generator(device=DEV).manual_seed(B * 7919 + n * 31 + D)
    m = torch.randn(B, D, device=DEV, generator=g)
    s = (torch.rand(B, D, device=DEV, generator=g) + 0.2) * sigma_scale
    X = torch.empty(B, n, D, device=DEV)
    ops.sample_batched(X, m, s, symmetric=False, seed=seed)
    return X, m, s


def _weights(B, n, active, seed):
    """Rank-assigned weights of fitnesses with a NaN in item 0 (the worst rank) and one zero weight per item."""
    st = sepcmaes(center_init=torch.zeros(4, device=DEV), stdev_init=1.0, objective_sense="min", popsize=n, active=active)
    g = torch.Generator(device=DEV).manual_seed(seed)
    f = torch.randn(B, n, device=DEV, generator=g)
    f[0, n // 2] = float("nan")
    aw = ops.rank_table_batched(f, False, st.weights)
    zero_row = (torch.arange(B, device=DEV) * 5 + 1) % n
    aw[torch.arange(B, device=DEV), zero_row] = 0.0
    return aw, zero_row


def _moments64(X, m, s, aw, active):
    D = X.shape[-1]
    z = (X.double() - m.double()[:, None, :]) / s.double()[:, None, :]
    awd = aw.double()
    a = awd.clamp_min(0.0)
    q = (z * z).sum(-1)
    b = torch.where(awd < 0, D * awd / q, awd) if active else awd
    return z, a, b


@pytest.mark.parametrize("active", [False, True])
@pytest.mark.parametrize("n", [2, 3, 7, 4097])
@pytest.mark.parametrize("D", [1, 3, 4, 5, 1025, 10_000])
def test_moments_batched_against_float64(D, n, active):
    """local, S2 and wsum of 3 items against float64 sums over the recovered steps, within the first-order bound of their fp32
    sums; stored == rebuilt bit for bit with the rows of zero weight poisoned with NaN (never read); item b == a one-item call on
    its own operands with stream_id0 = b, stored and rebuilt."""
    B, seed = 3, 1000 + D + n
    X, m, s = _population(B, n, D, seed)
    aw, zero_row = _weights(B, n, active, D + n)
    Xp = X.clone()
    Xp[torch.arange(B, device=DEV), zero_row] = float("nan")
    stored = ops.sepcma_moments_batched(Xp, m, s, aw, active)
    rebuilt = ops.sepcma_moments_batched(None, m, s, aw, active, seed=seed)
    for a, b in zip(stored, rebuilt):
        assert torch.equal(a, b)
    for b in range(B):
        one_s = ops.sepcma_moments_batched(Xp[b:b + 1], m[b:b + 1], s[b:b + 1], aw[b:b + 1], active)
        one_r = ops.sepcma_moments_batched(None, m[b:b + 1], s[b:b + 1], aw[b:b + 1], active, seed=seed, stream_id0=b)
        for full, x1, x2 in zip(stored, one_s, one_r):
            assert torch.equal(full[b:b + 1], x1) and torch.equal(x1, x2), b
    z, a, bw = _moments64(X, m, s, aw, active)
    local, S2, wsum = (t.double() for t in stored)
    zz, az = z * z, z.abs()
    ref_l, ref_s2, ref_w = torch.einsum("bn,bnd->bd", a, z), torch.einsum("bn,bnd->bd", bw, zz), bw.sum(-1)
    e_l = (gam(n) + 3 * EPS) * torch.einsum("bn,bnd->bd", a, az)
    rel_b = gam(n) + gam(D) + 16 * EPS  # the sums, q and the division that forms b
    e_s2 = rel_b * torch.einsum("bn,bnd->bd", bw.abs(), zz) + 1e-30
    e_w = rel_b * bw.abs().sum(-1) + 1e-30
    assert bool(((local - ref_l).abs() <= e_l + 1e-30).all()), float(((local - ref_l).abs() / (e_l + 1e-30)).max())
    assert bool(((S2 - ref_s2).abs() <= e_s2).all()), float(((S2 - ref_s2).abs() / e_s2).max())
    assert bool(((wsum - ref_w).abs() <= e_w).all())


def test_moments_batched_across_item_chunks():
    """70 000 items of 3 x 5: the stored and rebuilt sums agree bit for bit, items on both sides of the 65 535-item chunk edge
    equal one-item calls, and every item is within the float64 bound."""
    B, n, D, seed = 70_000, 3, 5, 77
    X, m, s = _population(B, n, D, seed)
    st = sepcmaes(center_init=torch.zeros(4, device=DEV), stdev_init=1.0, objective_sense="min", popsize=n)
    g = torch.Generator(device=DEV).manual_seed(3)
    aw = ops.rank_table_batched(torch.randn(B, n, device=DEV, generator=g), False, st.weights)
    stored = ops.sepcma_moments_batched(X, m, s, aw, True)
    rebuilt = ops.sepcma_moments_batched(None, m, s, aw, True, seed=seed)
    for a, b in zip(stored, rebuilt):
        assert torch.equal(a, b)
    for b in (0, 65_534, 65_535, 65_536, B - 1):
        one = ops.sepcma_moments_batched(None, m[b:b + 1], s[b:b + 1], aw[b:b + 1], True, seed=seed, stream_id0=b)
        for full, x1 in zip(stored, one):
            assert torch.equal(full[b:b + 1], x1), b
    z, a, bw = _moments64(X, m, s, aw, True)
    rel = gam(n) + gam(D) + 16 * EPS
    assert bool(((stored[0].double() - torch.einsum("bn,bnd->bd", a, z)).abs() <= rel * torch.einsum("bn,bnd->bd", a, z.abs()) + 1e-30).all())
    assert bool(((stored[1].double() - torch.einsum("bn,bnd->bd", bw, z * z)).abs()
                 <= rel * torch.einsum("bn,bnd->bd", bw.abs(), z * z) + 1e-30).all())


def _update_state(B, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda *shape: torch.randn(*shape, device=DEV, generator=g)  # noqa: E731
    u = lambda *shape: torch.rand(*shape, device=DEV, generator=g)  # noqa: E731
    sigma = u(B) * 0.5 + 0.5
    A = (u(B, D) + 0.5).sqrt()
    return dict(local=r(B, D) * 0.4, S2=u(B, D) * 1.8 + 0.2, wsum=u(B) * 0.5, m=r(B, D), p_sigma=r(B, D) * 0.3, p_c=r(B, D) * 0.1, sigma=sigma,
                C=u(B, D) + 0.5, A=A, s=sigma[:, None] * A)


@pytest.mark.parametrize("steps", [4, 5])
@pytest.mark.parametrize("bounds", [(None, None), (0.55, 0.8)])
@pytest.mark.parametrize("csa_squared", [False, True])
@pytest.mark.parametrize("D", [1, 1025, 3000])
def test_update_batched_equals_the_single_call(D, csa_squared, bounds, steps):
    """Every item of evok_sepcma_update_batched against evok_sepcma_update on that item's clones, bit for bit, on a generation
    that skips (steps 4) and one that takes (steps 5) the square root at decompose_C_freq 3, with and without stdev bounds."""
    B = 5
    st = sepcmaes(center_init=torch.zeros(D, device=DEV), stdev_init=1.0, objective_sense="min", popsize=12)
    consts = _consts(st.hyperparameters)
    t = _update_state(B, D, D + steps)
    batched = {k: v.clone() for k, v in t.items()}
    ops.sepcma_update_batched(batched["local"], batched["S2"], batched["wsum"], batched["m"], batched["p_sigma"], batched["p_c"], batched["sigma"],
                              batched["C"], batched["A"], batched["s"], consts, csa_squared, steps=steps, decompose_C_freq=3, stdev_min=bounds[0],
                              stdev_max=bounds[1])
    for b in range(B):
        one = {k: v[b].clone().reshape(-1) for k, v in t.items()}
        ops.sepcma_update(one["local"], one["S2"], one["wsum"], one["m"], one["p_sigma"], one["p_c"], one["sigma"], one["C"], one["A"], one["s"],
                          consts, csa_squared, decompose_C_freq=3, steps=steps, stdev_min=bounds[0], stdev_max=bounds[1])
        for k in ("m", "p_sigma", "p_c", "sigma", "C", "A", "s"):
            assert torch.equal(batched[k][b].reshape(-1), one[k]), (b, k)
    decomposed = (steps + 1) % 3 == 0
    assert torch.equal(batched["A"], batched["C"].sqrt()) == decomposed
    assert torch.equal(batched["A"], t["A"]) != decomposed


def _run(objective, B, n, D, generations, lazy, seed=5, **kw):
    torch.manual_seed(seed)
    g = torch.Generator(device=DEV).manual_seed(seed)
    st = sepcmaes(center_init=torch.rand(B, D, device=DEV, generator=g) * 4 - 2, stdev_init=torch.rand(B, device=DEV, generator=g) + 0.5,
                  objective_sense="min", popsize=n, **kw)
    states = []
    for _ in range(generations):
        values, evals = sepcmaes_ask_and_evaluate(st, objective=objective, lazy=lazy)
        assert isinstance(values, LazyPopulation) == lazy
        st = sepcmaes_tell(st, values, evals)
        states.append(st)
    return states


def _same_state(a, b):
    for k in ("center", "sigma", "C", "A", "s", "p_sigma", "p_c"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


@pytest.mark.parametrize("objective", ["rastrigin", "shifted_sphere"])
def test_lazy_runs_equal_stored_runs_bit_for_bit(objective):
    """Sample-and-evaluate stores the population `sepcmaes_ask` returns under the same seed, `materialize()` rebuilds it, and a lazy
    run and a stored run give bit-identical states over 12 generations: for a built-in objective, and for a FusedObjective with one
    shift per item (data batch shape = the state's)."""
    B, n, D = 24, 37, 131
    g = torch.Generator(device=DEV).manual_seed(9)
    obj = rastrigin if objective == "rastrigin" else FusedObjective("shifted_sphere", *SHIFTED_SPHERE,
                                                                  data={"o": torch.randn(B, D, device=DEV, generator=g)})
    st = _run(obj, B, n, D, 1, False, stdev_min=0.05)[0]
    torch.manual_seed(11)
    asked = sepcmaes_ask(st)
    torch.manual_seed(11)
    stored, f_stored = sepcmaes_ask_and_evaluate(st, objective=obj)
    torch.manual_seed(11)
    lazy, f_lazy = sepcmaes_ask_and_evaluate(st, objective=obj, lazy=True)
    assert torch.equal(asked, stored) and torch.equal(f_stored, f_lazy) and torch.equal(lazy.materialize(), stored)
    _same_state(sepcmaes_tell(st, stored, f_stored), sepcmaes_tell(st, lazy, f_lazy))
    a = _run(obj, B, n, D, 12, False, stdev_min=0.05)
    b = _run(obj, B, n, D, 12, True, stdev_min=0.05)
    for sa, sb in zip(a, b):
        _same_state(sa, sb)
    assert a[-1].generation == 12 and bool(torch.isfinite(a[-1].center).all())


@pytest.mark.parametrize("shape,kw", [((256, 20, 128), {}), ((256, 21, 128), dict(active=False, csa_squared=True)),
                                      ((64, 16, 96), dict(stdev_min=0.3, stdev_max=0.6)), ((4, 2000, 4096), {}),
                                      ((32, 12, 40), dict(c_1_ratio=0.05, c_mu_ratio=0.05))])
def test_generations_against_the_float64_reference(shape, kw):
    """Three generations (stored populations, the rastrigin kernel's fitnesses) of every item against the float64 reference fed
    that item's state, values and fitnesses, within the fp32 bound.  Repaired values: the last generation tells a population
    clipped to a box, whose steps differ from the drawn ones."""
    B, n, D = shape
    torch.manual_seed(21)
    g = torch.Generator(device=DEV).manual_seed(21)
    st = sepcmaes(center_init=torch.rand(B, D, device=DEV, generator=g) * 2 - 1, stdev_init=torch.rand(B, device=DEV, generator=g) * 0.3 + 0.4,
                  objective_sense="min", popsize=n, **kw)
    worst = 0.0
    for gen in range(3):
        values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin)
        if gen == 2:
            values = values.clamp(-1.0, 1.0)
            evals = rastrigin(values)
        new = sepcmaes_tell(st, values, evals)
        record = []
        ratios = SO.tell_ratios(st, values, evals, new, record=record)
        near = [b for b, r in enumerate(record) if abs(r["margin"]) < 1e-3]
        ok = [r for b, r in enumerate(ratios) if b not in near]
        assert len(ok) >= B - max(1, B // 50) and max(ok) <= 1.0, (gen, max(ok))
        worst = max(worst, max(ok))
        st = new
    print(f"{shape} {kw}: worst error / bound {worst:.3f}")


def test_launches_do_not_grow_with_the_batch():
    """A whole ask-evaluate-tell generation is the same number of launches at B = 1 and B = 300, stored and lazy."""
    counts = {}
    for B in (1, 300):
        for lazy in (False, True):
            st = sepcmaes(center_init=torch.zeros(B, 50, device=DEV), stdev_init=1.0, objective_sense="min", popsize=16)
            values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin, lazy=lazy)
            st = sepcmaes_tell(st, values, evals)  # warm
            before = ops.launch_count()
            values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin, lazy=lazy)
            sepcmaes_tell(st, values, evals)
            counts[B, lazy] = ops.launch_count() - before
    assert counts[1, False] == counts[300, False] and counts[1, True] == counts[300, True], counts
    assert counts[1, True] <= 6, counts  # sample + evaluate, rank table, q pass, column pass, its sums, update


def test_ask_and_tell_never_synchronise():
    torch.manual_seed(2)
    st = sepcmaes(center_init=torch.randn(16, 20, device=DEV), stdev_init=1.0, objective_sense="min", stdev_min=0.01, stdev_max=10.0)
    values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin, lazy=True)
    st = sepcmaes_tell(st, values, evals)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for lazy in (False, True):
            values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin, lazy=lazy)
            st = sepcmaes_tell(st, values, evals)
        x = sepcmaes_ask(st)
        st = sepcmaes_tell(st, x, rastrigin(x))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert st.generation == 4


def test_lazy_run_needs_no_population_memory():
    """16 x 1000 x 100 000 (6.4 GB if stored): a lazy generation allocates at most the next state, the moments and the workspaces
    on top of the state it starts from, a few per cent of the population."""
    B, n, D = 16, 1000, 100_000
    st = sepcmaes(center_init=torch.zeros(B, D, device=DEV), stdev_init=1.0, objective_sense="min", popsize=n)
    values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin, lazy=True)
    st = sepcmaes_tell(st, values, evals)
    del values, evals
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(2):
        values, evals = sepcmaes_ask_and_evaluate(st, objective=rastrigin, lazy=True)
        st = sepcmaes_tell(st, values, evals)
        del values, evals
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    state_bytes = 7 * B * D * 4
    print(f"peak above the starting state: {peak / 2**20:.1f} MiB (state {state_bytes / 2**20:.1f} MiB, population {B * n * D * 4 / 2**30:.1f} GiB)")
    assert peak < 2 * state_bytes + 64 * 2**20, peak
    assert math.isfinite(float(st.sigma.max()))
