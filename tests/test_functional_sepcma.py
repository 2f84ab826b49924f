"""The functional separable CMA-ES (`algorithms/functional/funcsepcmaes.py`) without a device: the float64 reference against the
reference's own separable run, the batched torch tell against that reference per item, the reference's mutations, the constants
against `CMAES(separable=True)`, argument errors, and the return codes of the two batched entry points on calls that return
before any device work."""

import functools
import os

import numpy as np
import pytest
import torch

from evotorch_b200 import Problem
from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200.algorithms import CMAES
from evotorch_b200.algorithms.functional import LazyPopulation, sepcmaes, sepcmaes_ask, sepcmaes_ask_and_evaluate, sepcmaes_tell
from evotorch_b200.objectives import FusedObjective
from oracle import functional_sepcma_oracle as SO

NULLPTR, BADSIZE, WORKSPACE = -1, -2, -4  # EVOK_E_* of include/evok.h
P = 64  # any non-null pointer: the argument checks never dereference it


def close(a, b, rtol, atol):
    np.testing.assert_allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=rtol, atol=atol)


def _torch_sphere(x):
    return torch.sum(x**2, dim=-1)


def test_oracle_reproduces_the_reference_separable_run():
    """The float64 reference, fed the values and fitnesses of the CPU op-by-op `CMAES(separable=True)` run, reproduces the
    reference's own separable run (tests/golden/cmaes_variants_golden.npz, "separable/*") for all 7 generations: steps recovered
    from the values give the reference's steps."""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "cmaes_variants_golden.npz"))
    prob = Problem("min", _torch_sphere, initial_bounds=(-3, 3), solution_length=8, vectorized=True, seed=11, dtype=torch.float32)
    c = CMAES(prob, stdev_init=1.0, popsize=14, separable=True)
    o = SO.item_state(sepcmaes(center_init=c.m.clone(), stdev_init=1.0, popsize=14, objective_sense="min"), 0)
    assert o.decompose_C_freq == c.decompose_C_freq
    for t in range(gold["separable/m"].shape[0]):
        c.step()
        SO.reference_generation(o, c.population.values.numpy(), c.population.evals[:, 0].numpy(), "min")
        close(c.population.evals[:, 0].numpy(), gold["separable/f"][t], rtol=2e-5, atol=2e-5)
        close(o.m, gold["separable/m"][t], rtol=2e-5, atol=5e-6)
        close(o.sigma, float(gold["separable/sigma"][t]), rtol=2e-5, atol=0)
        close(o.C, gold["separable/C"][t], rtol=5e-5, atol=5e-6)
        close(o.p_sigma, gold["separable/p_sigma"][t], rtol=5e-5, atol=5e-6)
        close(o.p_c, gold["separable/p_c"][t], rtol=5e-5, atol=5e-6)
    assert t == 6


# Batched float64 cases: items with different centres and step sizes, each with the options named.  "freq3" takes small learning
# rates so that limit_C_decomposition gives a decomposition every 3rd generation; "freq1" switches the limit off with the same
# rates.  "repaired" clips every population to a box after the draw, so recovered steps differ from the drawn ones.
CASES = {
    "plain": dict(batch=(3,), d=6, popsize=11, kw={}),
    "max_bounds": dict(batch=(2, 2), d=5, popsize=10, kw=dict(stdev_min=0.35, stdev_max=0.5), sense="max"),
    "csa_squared_inactive": dict(batch=(4,), d=7, popsize=12, kw=dict(csa_squared=True, active=False)),
    "freq3": dict(batch=(3,), d=12, popsize=9, kw=dict(c_1_ratio=0.024, c_mu_ratio=0.024, limit_C_decomposition=True)),
    "freq1": dict(batch=(3,), d=12, popsize=9, kw=dict(c_1_ratio=0.024, c_mu_ratio=0.024, limit_C_decomposition=False)),
    "repaired": dict(batch=(3,), d=8, popsize=13, kw={}, box=1.2),
}
GENERATIONS = 6


def _objective(x, sense):
    f = torch.sum(x**2 - 3 * torch.cos(2 * np.pi * x), dim=-1)
    return -f if sense == "max" else f


@functools.lru_cache(maxsize=None)
def _run(name):
    """The generations of a case on the torch path in float64: [(state, values, fitnesses, drawn z, told state), ...]."""
    case = CASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    batch, d = case["batch"], case["d"]
    center = torch.rand(batch + (d,), generator=g, dtype=torch.float64) * 2 - 1
    sigma = torch.rand(batch, generator=g, dtype=torch.float64) * 0.4 + 0.4
    sense = case.get("sense", "min")
    state = sepcmaes(center_init=center, stdev_init=sigma, popsize=case["popsize"], objective_sense=sense, **case["kw"])
    out = []
    for _ in range(GENERATIONS):
        z = torch.randn(batch + (state.popsize, d), generator=g, dtype=torch.float64)
        x = state.center[..., None, :] + state.s[..., None, :] * z
        if "box" in case:
            x = x.clamp(-case["box"], case["box"])
        f = _objective(x, sense)
        new = sepcmaes_tell(state, x, f)
        out.append((state, x, f, z, new))
        state = new
    return out


def test_case_options_hold():
    """Each case exercises what it is named for: decompositions every 3rd generation with the limit on and every generation with
    it off, an active stdev bound, and repaired values."""
    assert _run("freq3")[0][0].hyperparameters.decompose_C_freq == 3
    assert _run("freq1")[0][0].hyperparameters.decompose_C_freq == 1
    assert all(r[0].hyperparameters.decompose_C_freq == 1 for r in _run("plain"))
    stds = torch.stack([r[4].sigma[..., None] * r[4].C.sqrt() for r in _run("max_bounds")])
    assert bool(((stds - 0.35).abs() < 1e-12).any() or ((stds - 0.5).abs() < 1e-12).any())
    x, z, st = _run("repaired")[0][1], _run("repaired")[0][3], _run("repaired")[0][0]
    assert not torch.allclose(x, st.center[..., None, :] + st.s[..., None, :] * z)


@pytest.mark.parametrize("name", list(CASES))
def test_torch_tell_matches_the_float64_reference_per_item(name):
    """Every generation of every item of the batched float64 torch tell against the reference fed that item's state, values and
    fitnesses, within the float64 bound; h_sig is far from its threshold (the bound takes it as exact)."""
    for gen, (state, x, f, z, new) in enumerate(_run(name)):
        record = []
        ratios = SO.tell_ratios(state, x, f, new, record=record)
        assert max(ratios) <= 1.0, (gen, ratios)
        assert all(abs(r["margin"]) > 1e-9 for r in record)
        assert new.generation == state.generation + 1
        assert torch.equal(new.s, new.sigma[..., None] * new.A)


def test_every_mutation_is_rejected_by_some_case():
    """Each mutated reference is outside the bound on at least one item of one generation of one case, and the unmutated one
    is inside it on all of them: the cases above can tell the right algorithm from each wrong one."""
    worst = {m: 0.0 for m in SO.MUTATIONS}
    for name in CASES:
        for state, x, f, z, new in _run(name):
            for m in SO.MUTATIONS:
                worst[m] = max(worst[m], max(SO.tell_ratios(state, x, f, new, mutation=m, z_raw=z)))
    assert all(r > 10.0 for r in worst.values()), worst


def test_the_state_passed_in_is_left_unchanged():
    state, x, f, _, _ = _run("plain")[0]
    before = [t.clone() for t in (state.center, state.sigma, state.C, state.A, state.s, state.p_sigma, state.p_c)]
    sepcmaes_tell(state, x, f)
    for a, b in zip(before, (state.center, state.sigma, state.C, state.A, state.s, state.p_sigma, state.p_c)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kw", [dict(d=10), dict(d=33, popsize=20), dict(d=50, active=False), dict(d=7, c_1_ratio=0.5, c_mu_ratio=2.0),
                                dict(d=100, limit_C_decomposition=False), dict(d=16, c_sigma_ratio=0.7, damp_sigma_ratio=1.3, c_c_ratio=0.9, c_m=0.8)])
def test_constants_equal_the_separable_CMAES(kw):
    kw = dict(kw)
    d = kw.pop("d")
    prob = Problem("min", _torch_sphere, initial_bounds=(-1, 1), solution_length=d, vectorized=True, seed=0, dtype=torch.float32)
    c = CMAES(prob, stdev_init=0.5, separable=True, **kw)
    st = sepcmaes(center_init=torch.zeros(d), stdev_init=0.5, objective_sense="min", **kw)
    hp = st.hyperparameters
    assert hp.popsize == c.popsize and hp.mu == c.mu and hp.decompose_C_freq == c.decompose_C_freq
    assert torch.equal(hp.weights, c.weights)
    for name in ("mu_eff", "c_m", "c_sigma", "damp_sigma", "c_c", "c_1", "c_mu", "variance_discount_sigma", "variance_discount_c"):
        assert getattr(hp, name) == getattr(c, name), name
    assert hp.unbiased_expectation == c.unbiased_expectation and hp.weights_sum == c._weights_sum
    assert st.C.shape == st.A.shape == st.s.shape == (d,) and torch.equal(st.s, torch.full((d,), 0.5))


def test_batch_shapes_and_ask():
    st = sepcmaes(center_init=torch.zeros(2, 3, 5, dtype=torch.float64), stdev_init=torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64),
                  objective_sense="min", popsize=6)
    assert st.sigma.shape == (2, 3) and st.s.shape == (2, 3, 5) and torch.equal(st.s[:, 1], torch.full((2, 5), 0.2, dtype=torch.float64))
    x = sepcmaes_ask(st)
    assert x.shape == (2, 3, 6, 5) and x.dtype == torch.float64
    new = sepcmaes_tell(st, x, x.pow(2).sum(-1))
    assert new.center.shape == (2, 3, 5) and new.sigma.shape == (2, 3)


def test_argument_errors():
    st = sepcmaes(center_init=torch.zeros(2, 4), stdev_init=1.0, objective_sense="min", popsize=6)
    with pytest.raises(ValueError, match="per-item"):
        sepcmaes(center_init=torch.zeros(2, 4), stdev_init=1.0, objective_sense="min", c_m=torch.tensor([1.0, 0.5]))
    with pytest.raises(ValueError, match="per-item"):
        sepcmaes(center_init=torch.zeros(2, 4), stdev_init=1.0, objective_sense="min", stdev_min=torch.tensor([0.1, 0.2]))
    with pytest.raises(ValueError, match="objective_sense"):
        sepcmaes(center_init=torch.zeros(4), stdev_init=1.0, objective_sense="minimize")
    x = sepcmaes_ask(st)
    with pytest.raises(ValueError, match="`values`"):
        sepcmaes_tell(st, x[:, :5], torch.zeros(2, 5))
    with pytest.raises(ValueError, match="`values`"):
        sepcmaes_tell(st, x[0], torch.zeros(6))
    with pytest.raises(ValueError, match="`evals`"):
        sepcmaes_tell(st, x, torch.zeros(2, 5))
    with pytest.raises(ValueError, match="`evals`"):
        sepcmaes_tell(st, x, torch.zeros(6))
    other = sepcmaes(center_init=torch.zeros(2, 4), stdev_init=1.0, objective_sense="min", popsize=6)
    pop = LazyPopulation(torch.Size((2, 6, 4)), 1, 6, False, other.center, other.s)
    with pytest.raises(ValueError, match="another centre"):
        sepcmaes_tell(st, pop, torch.zeros(2, 6))
    told = sepcmaes_tell(st, x, x.pow(2).sum(-1))
    with pytest.raises(ValueError, match="another"):  # a population of this state, told to its successor
        sepcmaes_tell(told, LazyPopulation(torch.Size((2, 6, 4)), 1, 6, False, st.center, st.s), torch.zeros(2, 6))
    with pytest.raises(ValueError, match="lazy=True"):
        sepcmaes_ask_and_evaluate(st, objective=_torch_sphere, lazy=True)
    values, evals = sepcmaes_ask_and_evaluate(st, objective=_torch_sphere)
    assert values.shape == (2, 6, 4) and evals.shape == (2, 6)
    shifted = FusedObjective("shifted_sphere", {"s": "(x - o)**2"}, "s", data={"o": torch.zeros(3, 4)})
    with pytest.raises(ValueError, match="batch shape"):
        sepcmaes_ask_and_evaluate(st, objective=shifted)
    single = sepcmaes(center_init=torch.zeros(4), stdev_init=1.0, objective_sense="min", popsize=6)
    with pytest.raises(ValueError, match="batch shape"):  # a state of batch shape () is not broadcast to the data's items
        sepcmaes_ask_and_evaluate(single, objective=shifted)


# ------------------------------------------------------------------------------------------------ C ABI return codes
@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def _no_launch(lib, call):
    before = lib.evok_launch_count()
    rc = call()
    assert lib.evok_launch_count() == before
    return rc


# 2 items of 8 rows x 4 columns; with ws_bytes = 0 a valid call stops at EVOK_E_WORKSPACE
MOMENTS_BASE = dict(X=P, sx=32, ldx=4, m=P, s=P, aw=P, active=1, items=2, rows=8, D=4, local=P, S2=P, wsum=P, ws=P, ws_bytes=0)
MOMENTS_CASES = [
    ({}, WORKSPACE),
    (dict(X=None), WORKSPACE),  # lazy: the rows are rebuilt
    (dict(active=0), WORKSPACE),
    (dict(items=0), 0),
    (dict(items=0, X=None), 0),
    (dict(items=-1), BADSIZE),
    (dict(rows=0), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(ldx=3), BADSIZE),
    (dict(ldx=3, X=None), WORKSPACE),  # no rows are read: ldx is not used
    (dict(sx=-32), BADSIZE),
    (dict(m=None), NULLPTR),
    (dict(s=None), NULLPTR),
    (dict(aw=None), NULLPTR),
    (dict(local=None), NULLPTR),
    (dict(S2=None), NULLPTR),
    (dict(wsum=None), NULLPTR),
    (dict(ws=None), NULLPTR),
    (dict(m=None, items=0), NULLPTR),
    (dict(items=-1, ldx=3), BADSIZE),
]


def moments_call(lib, a):
    return lib.evok_sepcma_moments_batched(a["X"], a["sx"], a["ldx"], a["m"], a["s"], a["aw"], a["active"], a["items"], a["rows"], a["D"], 1, 0,
                                           a["local"], a["S2"], a["wsum"], a["ws"], a["ws_bytes"], None)


@pytest.mark.parametrize("changes,code", MOMENTS_CASES)
def test_sepcma_moments_batched_codes(lib, changes, code):
    assert _no_launch(lib, lambda: moments_call(lib, dict(MOMENTS_BASE, **changes))) == code


def test_sepcma_moments_batched_workspace_grows_with_the_items(lib):
    """At least one row chunk of partial sums per item of a chunk of at most 65 535 items, and q for every item."""
    for items, rows, D in ((1, 100, 64), (70000, 100, 64), (3, 4097, 1025), (1, 100000, 4096)):
        need = min(items, 65535) * 2 * D * 4 + items * rows * 4
        assert lib.evok_sepcma_moments_batched_workspace_bytes(items, rows, D) >= need
    assert lib.evok_sepcma_moments_batched_workspace_bytes(0, 100, 64) == 256


UPDATE_BASE = dict(local=P, S2=P, wsum=P, items=0, D=4, m=P, ps=P, pc=P, sigma=P, C=P, A=P, s=P, freq=1)
UPDATE_CASES = [
    ({}, 0),
    (dict(items=-1), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(freq=0), BADSIZE),
    (dict(local=None), NULLPTR),
    (dict(S2=None), NULLPTR),
    (dict(wsum=None), NULLPTR),
    (dict(m=None), NULLPTR),
    (dict(ps=None), NULLPTR),
    (dict(pc=None), NULLPTR),
    (dict(sigma=None), NULLPTR),
    (dict(C=None), NULLPTR),
    (dict(A=None), NULLPTR),
    (dict(s=None), NULLPTR),
    (dict(consts=None), NULLPTR),
]


def update_call(lib, a):
    consts = a.get("consts", (nat.c_float * 10)(*([0.5] * 10)))
    return lib.evok_sepcma_update_batched(a["local"], a["S2"], a["wsum"], a["items"], a["D"], a["m"], a["ps"], a["pc"], a["sigma"], a["C"], a["A"],
                                          a["s"], 0, consts, 0, a["freq"], float("nan"), float("nan"), None)


@pytest.mark.parametrize("changes,code", UPDATE_CASES)
def test_sepcma_update_batched_codes(lib, changes, code):
    assert _no_launch(lib, lambda: update_call(lib, dict(UPDATE_BASE, **changes))) == code
