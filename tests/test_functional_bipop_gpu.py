"""BIPOP restarts of the functional CMA-ES families on the H100: the BIPOP restart stage against the oracle (flags, regimes, tiers,
budgets and centres bit for bit, run_stdev within one float32 ulp), whole runs replayed from their stop flags, items independent of
the others' regimes, 70 000 items, max_popsize 8192, lazy separable runs equal to stored ones with NaN pad rows, no host
synchronisation, a launch count that does not depend on the regimes, and the share of items that reach the optimum of 10-D
Rastrigin and Rosenbrock."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import (bipop_ladder, cmaes, cmaes_ask_and_evaluate, restarts, restarts_tell, sepcmaes,
                                                 sepcmaes_ask_and_evaluate)
from evotorch_b200.algorithms.functional import funcrestarts
from evotorch_b200.objectives import rastrigin
from oracle import functional_bipop_oracle as BO
from oracle import functional_restart_oracle as RO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
POLICY = ("regime", "large_tier", "large_evaluations", "small_evaluations", "last_large_evaluations")


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _ladder(lam0: int, multiplier: float, N: int, d: int = 5, separable: bool = False):
    state = (sepcmaes if separable else cmaes)(center_init=torch.zeros(d, device=DEV), stdev_init=1.0, objective_sense="min", popsize=lam0)
    return bipop_ladder(state, multiplier, N)


def _near_integer(raw: float) -> bool:
    """A float64 lambda_s that lies within 1e-9 of an integer without being one: CUDA's and numpy's exp / log may floor it apart."""
    return raw != round(raw) and abs(raw - round(raw)) < 1e-9


def _stage(c: dict, lad, seed: int) -> dict:
    """ops.cma_restart_batched in its BIPOP form on a constructed case; returns its outputs as float64 / int numpy arrays."""
    t = lambda k: torch.tensor(c[k], dtype=torch.float32, device=DEV).contiguous()  # noqa: E731
    i = lambda k, dt=torch.int64: torch.tensor(c[k], dtype=dt, device=DEV).contiguous()  # noqa: E731
    sep, B = c["separable"], c["B"]
    C = t("c_diag") if sep else torch.diag_embed(t("c_diag")).contiguous()
    A = t("r_diag") if sep else torch.diag_embed(t("r_diag")).contiguous()
    s = (t("sigma")[:, None] * t("r_diag")).contiguous() if sep else None
    o = dict(m=t("m"), sigma=t("sigma"), p_sigma=t("p_sigma"), p_c=t("p_c"), C=C, A=A, s=s, history=t("history"), best_x=t("best_x"),
             best_f=t("best_f"), num_restarts=i("num_restarts"), steps=i("gen"), flags=torch.full((B,), -1, dtype=torch.int32, device=DEV),
             tier=i("tier", torch.int32), num_evaluations=i("num_evaluations"), regime=i("regime", torch.int32), large_tier=i("large_tier", torch.int32),
             large_evaluations=i("large_evaluations"), small_evaluations=i("small_evaluations"), last_large_evaluations=i("last_large_evaluations"),
             run_stdev=t("run_stdev"))
    ops.cma_restart_batched(sep, t("f"), t("X"), c["maximize"], o["steps"], o["m"], o["sigma"], o["p_sigma"], o["p_c"], o["C"], o["A"], o["s"],
                            o["history"], o["best_x"], o["best_f"], o["num_restarts"], o["flags"], t("sigma_def"), t("lb"), t("ub"), c["thresholds"],
                            seed=seed, tier=o["tier"], tier_counts=lad.counts, tier_history=lad.history, num_evaluations=o["num_evaluations"],
                            **{k: o[k] for k in POLICY + ("run_stdev",)}, n_large=lad.n_large, popsize0=lad.popsizes[0])
    return {k: (v.double() if v.is_floating_point() else v).cpu().numpy() for k, v in o.items() if v is not None}


def _ulp_close(a: float, b: float) -> bool:
    return abs(a - b) <= float(np.spacing(np.float32(max(abs(a), abs(b)))))


# ------------------------------------------------------------------------------------------------ the stage
@pytest.mark.parametrize("separable", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
@pytest.mark.parametrize("multiplier", [2.0, 1.5])
def test_restart_bipop_against_oracle(separable, maximize, multiplier):
    c = BO.constructed_bipop_items(separable, maximize, multiplier=multiplier)
    lad = _ladder(6, multiplier, 16, c["D"], separable)
    assert list(lad.popsizes) == c["sizes"]
    seed = 0x1357_9BDF_2468
    o = _stage(c, lad, seed)
    u_pol = BO.bipop_uniforms(seed, c["B"])
    exp = BO.expected(c, RO.reset_uniforms(seed, c["B"], c["D"]), u_pol, float32=True)
    for b, e in enumerate(exp):
        assert o["flags"][b] == e["flags"], (b, o["flags"][b], e["flags"])
        np.testing.assert_array_equal(o["best_x"][b], e["best_x"])
        assert o["best_f"][b] == e["best_f"]
        np.testing.assert_array_equal(o["history"][b], e["history"])
        for k in ("tier", "num_evaluations") + POLICY:
            assert o[k][b] == e[k], (b, k, o[k][b], e[k])
        assert o["steps"][b] == e["gen"] and o["num_restarts"][b] == e["num_restarts"]
        assert _ulp_close(o["run_stdev"][b], e["run_stdev"]), (b, o["run_stdev"][b], e["run_stdev"])
        if e["reset"]:
            np.testing.assert_array_equal(o["m"][b], e["centre"])
            assert o["sigma"][b] == o["run_stdev"][b]
            if separable:
                assert (o["s"][b] == o["run_stdev"][b]).all()
        else:
            np.testing.assert_array_equal(o["m"][b], c["m"][b])
    assert exp[5]["flags"] == 32 | 128 and exp[8]["flags"] == 128 and exp[10]["flags"] == 4


def test_restart_bipop_70000_items_and_small_popsizes():
    """Every item of 70 000 restarts (max_generations), across the 65 535 item chunk edge, from random policy states on the
    ladder 10 .. 8192: tiers (lambda_s up to 4096), budgets and regimes equal the oracle's, run_stdev within one ulp, and the
    centres of items on both sides of the edge equal the reset draw."""
    B, D = 70_000, 3
    lad = _ladder(10, 2, 8192, D)
    K, sizes = lad.n_large, list(lad.popsizes)
    rng = np.random.default_rng(4)
    regime = rng.integers(0, 3, B)
    lt = rng.integers(0, K, B)
    small_lam = rng.integers(10, 4097, B)
    tier = np.where(regime == 2, K + small_lam - 10, np.where(regime == 1, lt, 0))
    n_l, n_s = rng.integers(0, 5000, B), rng.integers(0, 5000, B)
    n_last = rng.integers(0, 100_000, B)
    sdef = rng.uniform(0.1, 3.0, B).astype(np.float32)
    gen = rng.integers(1, 4, B)
    thresholds = (None, None, None, None, None, 1.0)  # max_generations 1: every item restarts
    f = torch.zeros(B, 8192, device=DEV)
    i = lambda a, dt=torch.int64: torch.tensor(a, dtype=dt, device=DEV)  # noqa: E731
    z = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    o = dict(tier=i(tier, torch.int32), num_evaluations=i(np.zeros(B)), regime=i(regime, torch.int32), large_tier=i(lt, torch.int32), large_evaluations=i(n_l),
             small_evaluations=i(n_s), last_large_evaluations=i(n_last), run_stdev=torch.tensor(sdef, device=DEV), steps=i(gen),
             m=z(B, D), flags=torch.empty(B, dtype=torch.int32, device=DEV))
    seed = 77
    ops.cma_restart_batched(True, f, None, False, o["steps"], o["m"], z(B) + 1, z(B, D), z(B, D), z(B, D) + 1, z(B, D) + 1, z(B, D), z(B, 20),
                            z(B, D), z(B) + math.inf, torch.zeros(B, dtype=torch.int64, device=DEV), o["flags"], torch.tensor(sdef, device=DEV),
                            z(B, D) - 1, z(B, D) + 1, thresholds, seed=seed, m_draw=z(B, D), s_draw=z(B, D), tier=o["tier"], tier_counts=lad.counts,
                            tier_history=lad.history, num_evaluations=o["num_evaluations"], **{k: o[k] for k in POLICY + ("run_stdev",)}, n_large=K,
                            popsize0=10)
    got = {k: v.cpu().numpy() for k, v in o.items()}
    u = BO.bipop_uniforms(seed, B)
    near = 0
    for b in range(B):
        n = sizes[tier[b]]
        nl, ns = BO.account(int(regime[b]), n, int(n_l[b]), int(n_s[b]))
        assert got["flags"][b] == 32 | BO.budget_bit(int(regime[b]), int(gen[b]), n, int(n_last[b])), b
        e = BO.next_run(sizes=sizes, K=K, regime=int(regime[b]), large_tier=int(lt[b]), tier=int(tier[b]), gen=int(gen[b]), n=n, large_evaluations=nl,
                        small_evaluations=ns, last_large_evaluations=int(n_last[b]), sigma_def=float(sdef[b]), u=u[b], float32=True)
        assert (got["large_evaluations"][b], got["small_evaluations"][b], got["num_evaluations"][b]) == (nl, ns, n), b
        for k in ("regime", "large_tier", "last_large_evaluations"):
            assert got[k][b] == e[k], (b, k)
        if e["small_popsize"] is not None and _near_integer(BO.small_popsize_raw(10, sizes[int(lt[b])], u[b][0])):
            near += 1
        else:
            assert got["tier"][b] == e["tier"], (b, got["tier"][b], e["tier"])
        assert _ulp_close(float(got["run_stdev"][b]), e["run_stdev"]), b
    assert near <= 3, near
    small = got["regime"] == 2
    lam = np.array(sizes)[got["tier"][small]]
    assert lam.min() == 10 and lam.max() > 3000 and lam.max() <= 4096
    rows = [0, 65_534, 65_535, 65_536, B - 1]
    np.testing.assert_array_equal(got["m"][rows], RO.centre(-1.0, 1.0, RO.reset_uniforms(seed, B, D)[rows], True))


# ------------------------------------------------------------------------------------------------ whole runs
def _run(family: str, gens: int, B: int, d: int, lazy: bool = False, pad_nan: bool = False, seed: int = 5, setup=None, max_popsize: int = 40):
    """A BIPOP run from popsize 5 (x2, max `max_popsize`); returns the states after every tell and the seed of every restart stage."""
    torch.manual_seed(seed)
    make = cmaes if family == "cmaes" else sepcmaes
    state = make(center_init=torch.rand(B, d, device=DEV) * 10 - 5, stdev_init=2.0, objective_sense="min", popsize=5)
    rs = restarts(state, lb=-5.0, ub=5.0, max_generations=4, min_fitness_stdev=1e-3, popsize_multiplier=2, max_popsize=max_popsize, bipop=True)
    if setup is not None:
        rs = setup(rs)
    out, seeds = [], []
    draw = funcrestarts.draw_philox_seed

    def record():
        seeds.append(draw())
        return seeds[-1]

    funcrestarts.draw_philox_seed = record
    try:
        for _ in range(gens):
            if family == "cmaes":
                values, evals = cmaes_ask_and_evaluate(rs.search, objective=rastrigin)
            else:
                values, evals = sepcmaes_ask_and_evaluate(rs.search, objective=rastrigin, lazy=lazy)
            if pad_nan:
                pad = torch.arange(max_popsize, device=DEV) >= rs.popsize[:, None]
                values = torch.where(pad[:, :, None], math.nan, values)
                evals = torch.where(pad, math.nan, evals)
            rs = restarts_tell(rs, values, evals)
            out.append(rs)
    finally:
        funcrestarts.draw_philox_seed = draw
    return out, seeds


def _all(rs) -> list:
    return [_bits(t) for t in list(rs.search) + list(rs) if isinstance(t, torch.Tensor)]


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 33, 130])
def test_runs_replay_from_their_flags(family, d):
    """The regimes, tiers, budgets and run_stdev of every tell of a run equal those `replay` derives from the stop flags and each
    stage's draw, and bit 7 is set exactly where the replayed policy puts it."""
    B, G = 7, 40
    states, seeds = _run(family, G, B, d)
    flags = np.stack([s.stop_flags.cpu().numpy() for s in states])
    lad = states[0].ladder
    u = np.stack([BO.bipop_uniforms(s, B) for s in seeds])
    rep = BO.replay(flags, u, sizes=list(lad.popsizes), K=lad.n_large, sigma_def=np.full(B, 2.0), float32=True)
    near = 0
    for g, s in enumerate(states):
        np.testing.assert_array_equal(flags[g] & 128, rep["budget"][g], err_msg=str(g))
        for k in POLICY + ("num_evaluations",):
            np.testing.assert_array_equal(getattr(s, k).cpu().numpy(), rep[k][g], err_msg=f"{g} {k}")
        np.testing.assert_array_equal(s.item_generation.cpu().numpy(), rep["gen"][g])
        tier = s.tier.cpu().numpy()
        for b in range(B):
            if tier[b] != rep["tier"][g, b]:
                near += 1  # allowed only where lambda_s lies within 1e-9 of an integer
                lt = int(rep["large_tier"][g, b])
                assert _near_integer(BO.small_popsize_raw(5, lad.popsizes[lt], u[g, b, 0])), (g, b)
        for b in range(B):
            assert _ulp_close(float(s.run_stdev[b]), rep["run_stdev"][g, b]), (g, b)
    assert near <= 1
    assert {0, 1, 2} <= set(rep["regime"].ravel().tolist()) and (flags & 128).any()
    assert (rep["tier"] > lad.n_large).any()  # a small run above lambda_0


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 33, 130])
def test_items_do_not_depend_on_the_others_regimes(family, d):
    """Item 0 in a small run, in a batch of mixed regimes, equals item 0 of a batch where every item is in that small run."""
    B = 5

    def policy(regimes, n_l):
        def setup(rs):
            K = rs.ladder.n_large
            reg = torch.tensor(regimes, dtype=torch.int32, device=DEV)
            tier = torch.where(reg == 2, K + 3, torch.where(reg == 1, 2, 0)).to(torch.int32)
            return rs._replace(regime=reg, tier=tier, large_tier=torch.where(reg == 0, 0, 2).to(torch.int32), large_evaluations=torch.tensor(n_l, device=DEV),
                               small_evaluations=torch.full((B,), 10, device=DEV), last_large_evaluations=torch.full((B,), 60, device=DEV),
                               run_stdev=torch.full((B,), 0.3, device=DEV))
        return setup

    a, _ = _run(family, 6, B, d, seed=7, setup=policy([2, 0, 1, 2, 1], [300, 0, 40, 7, 500]))
    b, _ = _run(family, 6, B, d, seed=7, setup=policy([2] * B, [300] * B))
    for ra, rb in zip(a, b):
        for x, y in zip(_all(ra), _all(rb)):
            if x.ndim and x.shape[0] == B:
                assert torch.equal(x[0], y[0])


def test_lazy_separable_equals_stored_with_nan_pad_rows():
    (stored, _), (lazy, _) = _run("sepcmaes", 16, 9, 40, pad_nan=True), _run("sepcmaes", 16, 9, 40, lazy=True)
    for a, b in zip(stored, lazy):
        for x, y in zip(_all(a), _all(b)):
            assert torch.equal(x, y)
    assert any(bool((s.regime == 2).any()) for s in stored) and not stored[-1].best_values.isnan().any()


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
def test_max_popsize_8192(family):
    """Items in small runs of up to 4096 rows on the ladder 10 .. 8192: whole generations run, and the item at lambda_s = 4096
    tells only its first 4096 rows."""
    B, d = 3, 4

    def setup(rs):
        K = rs.ladder.n_large
        lam = torch.tensor([4096, 10, 2000], device=DEV)
        return rs._replace(regime=torch.full((B,), 2, dtype=torch.int32, device=DEV), tier=(K + lam - 10).to(torch.int32),
                           large_tier=torch.full((B,), K - 1, dtype=torch.int32, device=DEV), large_evaluations=torch.full((B,), 10**6, device=DEV),
                           last_large_evaluations=torch.full((B,), 10**6, device=DEV), run_stdev=torch.full((B,), 0.5, device=DEV))

    torch.manual_seed(1)
    make, ask = (cmaes, cmaes_ask_and_evaluate) if family == "cmaes" else (sepcmaes, sepcmaes_ask_and_evaluate)
    state = make(center_init=torch.rand(B, d, device=DEV), stdev_init=1.0, objective_sense="min", popsize=10)
    rs = setup(restarts(state, lb=-5.0, ub=5.0, max_generations=2, popsize_multiplier=2, max_popsize=8192, bipop=True))
    assert rs.search.popsize == 8192 and rs.popsize.tolist() == [4096, 10, 2000]
    for _ in range(3):
        values, evals = ask(rs.search, objective=rastrigin)
        pad = torch.arange(8192, device=DEV) >= rs.popsize[:, None]
        rs = restarts_tell(rs, values, torch.where(pad, math.nan, evals))
        assert torch.isfinite(rs.best_evals).all() and torch.isfinite(rs.search.center).all()
    assert (rs.num_evaluations == 2 * torch.tensor([4096, 10, 2000], device=DEV) + rs.popsize).all()
    assert int(rs.ladder.popsizes[-1]) == 4096 and rs.ladder.weights.shape == (rs.ladder.n_large + 4087, 8192)


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
def test_no_host_synchronisation_and_launch_count(family):
    torch.manual_seed(0)
    make = cmaes if family == "cmaes" else sepcmaes
    ask = cmaes_ask_and_evaluate if family == "cmaes" else sepcmaes_ask_and_evaluate
    rs = restarts(make(center_init=torch.randn(33, 9, device=DEV), stdev_init=1.0, objective_sense="min", popsize=6), lb=-3.0, ub=3.0,
                  max_generations=2, min_fitness_stdev=1e-6, popsize_multiplier=2, max_popsize=48, bipop=True)
    pops = []
    for _ in range(6):
        pops.append(ask(rs.search, objective=rastrigin))
        rs = restarts_tell(rs, *pops[-1])
    torch.cuda.synchronize()
    counts, regimes = [], []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for values, evals in pops:
            regimes.append(rs.regime.clone())
            before = ops.launch_count()
            rs = restarts_tell(rs, values, evals)
            counts.append(ops.launch_count() - before)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(set(counts)) == 1, counts
    assert len({tuple(t.tolist()) for t in regimes}) > 1  # the mix of regimes changed between the counted generations


# ------------------------------------------------------------------------------------------------ what BIPOP buys
def _rosenbrock(x: torch.Tensor) -> torch.Tensor:
    return (100.0 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1.0 - x[..., :-1]) ** 2).sum(-1)


def _share(objective, B: int, gens: int, bound: float, tol_fun: float, bipop: bool) -> tuple:
    torch.manual_seed(123)
    state = cmaes(center_init=torch.rand(B, 10, device=DEV) * 2 * bound - bound, stdev_init=0.3 * bound, objective_sense="min", popsize=10)
    rs = restarts(state, lb=-bound, ub=bound, tol_fun=tol_fun, popsize_multiplier=2, max_popsize=640, bipop=bipop)
    for _ in range(gens):
        values, evals = cmaes_ask_and_evaluate(rs.search, objective=objective)
        rs = restarts_tell(rs, values, evals)
    return (rs.best_evals < 1e-8).float().mean().item(), rs.num_evaluations.double().mean().item(), rs.best_evals.isnan().any().item()


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
def test_bipop_reaches_the_optimum(name):
    objective = rastrigin if name == "rastrigin" else _rosenbrock
    bound = 5.12 if name == "rastrigin" else 5.0
    tol_fun = 1e-4 if name == "rastrigin" else 1e-12  # as in the IPOP test
    gens = 2000
    bipop, bipop_evals, nan = _share(objective, 512, gens, bound, tol_fun, True)
    ipop, ipop_evals, _ = _share(objective, 512, gens, bound, tol_fun, False)
    print(f"{name} 10-D, 512 items x {gens} generations, share with f < 1e-8: BIPOP from 10 (x2, max 640) {bipop:.3f} at {bipop_evals:.0f} "
          f"evaluations per item; IPOP {ipop:.3f} at {ipop_evals:.0f}")
    assert not nan
    # measured on an H100 80GB HBM3 at 700 W: Rastrigin 0.070 at 39 592 evaluations per item (IPOP: 1.000 at 791 675), Rosenbrock
    # 0.932 at 20 200 (IPOP: 0.932 at 20 200; tol_fun 1e-12 rarely fires there).  The floors sit below those shares by 0.04 and
    # 0.08; BIPOP's small runs keep its evaluations per generation well below IPOP's on Rastrigin.
    if name == "rastrigin":
        assert bipop > 0.03 and bipop_evals < ipop_evals / 4
    else:
        assert bipop > 0.85
