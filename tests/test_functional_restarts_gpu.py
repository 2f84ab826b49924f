"""Restarts of the functional CMA-ES families on the H100: the restart stage against the float64 oracle (flags, best values and
centres bit for bit), whole runs with forced restarts against fresh searches and one-item tells at each item's own counter,
lazy separable runs equal to stored ones, isolation of items, no host synchronisation, and the share of items that reach the
global optimum with and without restarts."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask_and_evaluate, cmaes_tell, restarts, restarts_tell, sepcmaes,
                                                 sepcmaes_ask_and_evaluate, sepcmaes_tell)
from evotorch_b200.objectives import rastrigin
from oracle import functional_restart_oracle as RO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _stage(c: dict, seed: int, lazy: bool = False) -> dict:
    """The restart stage on a constructed case, float32 on the device; returns every output as numpy (float64 / int)."""
    t = lambda k: torch.tensor(c[k], dtype=torch.float32, device=DEV).contiguous()  # noqa: E731
    B, D, N = c["B"], c["D"], c["N"]
    sep = c["separable"]
    C = t("c_diag") if sep else torch.diag_embed(t("c_diag")).contiguous()
    A = t("r_diag") if sep else torch.diag_embed(t("r_diag")).contiguous()
    s = (t("sigma")[:, None] * t("r_diag")).contiguous() if sep else None
    out = dict(m=t("m"), sigma=t("sigma"), p_sigma=t("p_sigma"), p_c=t("p_c"), C=C, A=A, s=s, history=t("history"), best_x=t("best_x"), best_f=t("best_f"),
               num_restarts=torch.tensor(c["num_restarts"], device=DEV), steps=torch.tensor(c["gen"], device=DEV),
               flags=torch.full((B,), -1, dtype=torch.int32, device=DEV))
    X, draw = t("X"), {}
    if lazy:
        m_draw, s_draw = t("m") + 0.25, t("p_sigma").abs() + 0.5
        X = torch.empty(B, N, D, device=DEV)
        ops.sample_batched(X, m_draw, s_draw, symmetric=False, seed=4242)
        draw = dict(m_draw=m_draw, s_draw=s_draw, draw_seed=4242)
        c["rows"] = X.double().cpu().numpy()
    ops.cma_restart_batched(sep, t("f"), None if lazy else X, c["maximize"], out["steps"], out["m"], out["sigma"], out["p_sigma"], out["p_c"], out["C"],
                            out["A"], out["s"], out["history"], out["best_x"], out["best_f"], out["num_restarts"], out["flags"], t("sigma0"), t("lb"),
                            t("ub"), c["thresholds"], seed=seed, **draw)
    torch.cuda.synchronize()
    return {k: (v.double() if v.is_floating_point() else v).cpu().numpy() for k, v in out.items() if v is not None}


@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("separable", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
def test_stage_against_oracle(separable, maximize, lazy):
    if lazy and not separable:
        pytest.skip("only the separable family rebuilds rows")
    c = RO.constructed_items(separable, maximize, D=7, N=9)
    seed = 0x1234_5678_9ABC
    o = _stage(c, seed, lazy)
    exp = RO.expected(c, RO.reset_uniforms(seed, c["B"], c["D"]), float32=True)
    D = c["D"]
    for b, e in enumerate(exp):
        assert o["flags"][b] == e["flags"], (b, o["flags"][b], e["flags"])
        np.testing.assert_array_equal(o["best_x"][b], e["best_x"])
        assert o["best_f"][b] == e["best_f"] or (math.isnan(o["best_f"][b]) and math.isnan(e["best_f"]))
        np.testing.assert_array_equal(o["history"][b], e["history"])
        assert o["steps"][b] == e["gen"] and o["num_restarts"][b] == e["num_restarts"]
        if e["reset"]:
            np.testing.assert_array_equal(o["m"][b], e["centre"])
            assert o["sigma"][b] == np.float32(c["sigma0"][b])
            assert not o["p_sigma"][b].any() and not o["p_c"][b].any()
            one = np.ones(D) if separable else np.eye(D)
            np.testing.assert_array_equal(o["C"][b], one)
            np.testing.assert_array_equal(o["A"][b], one)
            if separable:
                np.testing.assert_array_equal(o["s"][b], np.full(D, np.float32(c["sigma0"][b])))
            assert (o["m"][b] >= c["lb"][b]).all() and (o["m"][b] <= c["ub"][b]).all()
        else:
            np.testing.assert_array_equal(o["m"][b], c["m"][b])
    for b, bit in RO.DESIGNED.items():
        assert o["flags"][b] & bit
    assert o["flags"][0] == 0


def _tensors(rs) -> list:
    """Every tensor of a RestartState and of its search, floats as their bits (NaN payloads included)."""
    ts = [t for t in list(rs.search) + list(rs) if isinstance(t, torch.Tensor)]
    return [t.view(torch.int32) if t.dtype == torch.float32 else t for t in ts]


def _one_item(state, b: int, generation: int):
    fields = {k: getattr(state, k)[b:b + 1] for k in state._fields if isinstance(getattr(state, k), torch.Tensor)}
    return state._replace(generation=generation, **fields)


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 33, 130])
def test_core_invariant_with_forced_restarts(family, d):
    """Every generation: a restarted item is bit-identical to a fresh search at its new centre; every other item has the state the
    family's tell gives its one-item state at its own counter (bit for bit; for cmaes the Cholesky factor at float32 rounding)."""
    torch.manual_seed(11)
    B = 7 if d < 130 else 5
    full = family == "cmaes"
    make = cmaes if full else sepcmaes
    state = make(center_init=torch.rand(B, d, device=DEV) * 4 - 2, stdev_init=torch.linspace(0.5, 1.5, B, device=DEV), objective_sense="min")
    rs = restarts(state, lb=-2.0, ub=torch.linspace(1.0, 3.0, d, device=DEV), max_generations=3 if d < 130 else 2)
    sigma0 = state.sigma.clone()
    keys = ("center", "sigma", "C", "A", "p_sigma", "p_c") + (() if full else ("s",))
    restarted = 0
    for g in range(7):
        if full:
            values, evals = cmaes_ask_and_evaluate(rs.search, objective=rastrigin)
        else:
            values, evals = sepcmaes_ask_and_evaluate(rs.search, objective=rastrigin)
        gens = rs.item_generation.tolist()
        nxt = restarts_tell(rs, values, evals)
        flags = nxt.stop_flags.tolist()
        for b in range(B):
            if flags[b]:
                restarted += 1
                fresh = make(center_init=nxt.search.center[b:b + 1].clone(), stdev_init=sigma0[b:b + 1], objective_sense="min")
                assert nxt.item_generation[b].item() == 0
                for k in keys:
                    assert torch.equal(getattr(nxt.search, k)[b:b + 1], getattr(fresh, k)), (g, b, k)
            else:
                one = (cmaes_tell if full else sepcmaes_tell)(_one_item(rs.search, b, gens[b]), values[b:b + 1], evals[b:b + 1])
                assert nxt.item_generation[b].item() == gens[b] + 1
                for k in keys:
                    got, want = getattr(nxt.search, k)[b:b + 1], getattr(one, k)
                    if full and k == "A":
                        torch.testing.assert_close(got, want, rtol=4e-6, atol=1e-7)
                    else:
                        assert torch.equal(got, want), (g, b, k)
        rs = nxt
    assert restarted >= B


def _sep_run(lazy: bool, gens: int, B: int = 9, d: int = 40):
    torch.manual_seed(5)
    state = sepcmaes(center_init=torch.rand(B, d, device=DEV) * 10 - 5, stdev_init=2.0, objective_sense="min")
    rs = restarts(state, lb=-5.0, ub=5.0, max_generations=4, min_fitness_stdev=1e-3)
    out = []
    for _ in range(gens):
        values, evals = sepcmaes_ask_and_evaluate(rs.search, objective=rastrigin, lazy=lazy)
        rs = restarts_tell(rs, values, evals)
        out.append(rs)
    return out


def test_lazy_separable_equals_stored():
    stored, lazy = _sep_run(False, 12), _sep_run(True, 12)
    for a, b in zip(stored, lazy):
        for x, y in zip(_tensors(a), _tensors(b)):
            assert torch.equal(x, y)
    assert stored[-1].num_restarts.sum() > 0 and not stored[-1].best_values.isnan().any()


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("poison", ["nan_evals", "inf_evals", "nan_values", "inf_values"])
def test_isolation_of_items(family, poison):
    torch.manual_seed(2)
    B, d, k = 6, 12, 3
    make = cmaes if family == "cmaes" else sepcmaes
    rs = restarts(make(center_init=torch.randn(B, d, device=DEV), stdev_init=1.0, objective_sense="min"), lb=-3.0, ub=3.0, max_generations=5)
    ask = cmaes_ask_and_evaluate if family == "cmaes" else sepcmaes_ask_and_evaluate
    for _ in range(3):
        values, evals = ask(rs.search, objective=rastrigin)
        rs = restarts_tell(rs, values, evals)
    values, evals = ask(rs.search, objective=rastrigin)
    v2, e2 = values.clone(), evals.clone()
    bad = math.nan if poison.startswith("nan") else math.inf
    if poison.endswith("evals"):
        e2[k, ::2] = bad
    else:
        v2[k, 1, ::3] = bad
        e2[k, 1] = bad
    torch.manual_seed(9)
    clean = restarts_tell(rs, values, evals)
    torch.manual_seed(9)
    dirty = restarts_tell(rs, v2, e2)
    others = [b for b in range(B) if b != k]
    for x, y in zip(_tensors(clean), _tensors(dirty)):
        assert torch.equal(x[others], y[others])
    if poison == "nan_values":
        assert dirty.stop_flags[k].item() & 64


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
def test_no_host_synchronisation(family):
    torch.manual_seed(0)
    make = cmaes if family == "cmaes" else sepcmaes
    ask = cmaes_ask_and_evaluate if family == "cmaes" else sepcmaes_ask_and_evaluate
    rs = restarts(make(center_init=torch.randn(33, 9, device=DEV), stdev_init=1.0, objective_sense="min"), lb=-3.0, ub=3.0, max_generations=2,
                  min_fitness_stdev=1e-6)
    pops = []
    for _ in range(5):
        pops.append(ask(rs.search, objective=rastrigin))
        rs = restarts_tell(rs, *pops[-1])  # warm-up: module loads and library plans
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for values, evals in pops:
            rs = restarts_tell(rs, values, evals)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert rs.num_restarts.sum().item() > 0


def _rosenbrock(x: torch.Tensor) -> torch.Tensor:
    return (100.0 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1.0 - x[..., :-1]) ** 2).sum(-1)


def _share_at_optimum(objective, restart: bool, B: int, gens: int, bound: float, tol_fun: float, popsize: int) -> tuple:
    torch.manual_seed(123)
    state = cmaes(center_init=torch.rand(B, 10, device=DEV) * 2 * bound - bound, stdev_init=0.3 * bound, objective_sense="min", popsize=popsize)
    if restart:
        rs = restarts(state, lb=-bound, ub=bound, tol_fun=tol_fun)
        for _ in range(gens):
            values, evals = cmaes_ask_and_evaluate(rs.search, objective=objective)
            rs = restarts_tell(rs, values, evals)
        best = rs.best_evals
    else:
        best = torch.full((B,), math.inf, device=DEV)
        for _ in range(gens):
            values, evals = cmaes_ask_and_evaluate(state, objective=objective)
            state = cmaes_tell(state, values, evals)
            best = torch.minimum(best, torch.where(evals.isnan(), math.inf, evals).amin(-1))
    return (best < 1e-8).float().mean().item(), best.isnan().any().item()


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
def test_restarts_reach_the_optimum_more_often(name):
    objective = rastrigin if name == "rastrigin" else _rosenbrock
    bound = 5.12 if name == "rastrigin" else 5.0
    # the built-in Rastrigin sums to ~10 D in float32 (ulp(100) = 7.6e-6): a flat fitness range is 1e-4 there, not 1e-12; at the
    # default popsize of 10 a run almost never finds its global minimum (none of 9000 runs did), at 100 a fair share does
    tol_fun, popsize = (1e-4, 100) if name == "rastrigin" else (1e-12, None)
    with_r, nan_r = _share_at_optimum(objective, True, 512, 2000, bound, tol_fun, popsize)
    without, _ = _share_at_optimum(objective, False, 512, 2000, bound, tol_fun, popsize)
    print(f"{name} 10-D, popsize {popsize or 10}, 512 items x 2000 generations: share with f < 1e-8: with restarts {with_r:.3f}, "
          f"without {without:.3f}")
    assert not nan_r
    assert with_r > without
