"""BIPOP restarts of the functional CMA-ES families without a GPU: the tables against the default constants of every population
size, argument validation, the torch restart stage against the float64 oracle in every branch of the regime policy, a hand-worked
schedule of regimes, tiers and budgets, whole float64 runs checked item by item against one-item searches of the item's
population size and step size, and the return codes of the BIPOP C entry point on calls that launch nothing."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import (bipop_ladder, cmaes, cmaes_ask, cmaes_tell, ipop_ladder, restarts, restarts_tell, sepcmaes,
                                                 sepcmaes_ask, sepcmaes_tell)
from evotorch_b200.algorithms.functional.funccmaes import _consts
from evotorch_b200.algorithms.functional.funcrestarts import BIPOP_FIELDS, _restart_torch
from oracle import functional_bipop_oracle as BO

NULLPTR, BADSIZE = -1, -2
P = 64  # any non-null pointer: the argument checks never dereference it
FAMILIES = {"cmaes": (cmaes, cmaes_ask, cmaes_tell), "sepcmaes": (sepcmaes, sepcmaes_ask, sepcmaes_tell)}
FIELDS = ("center", "sigma", "C", "A", "p_sigma", "p_c")


def _state(family: str, B: int = 4, d: int = 3, popsize: int = 10, **kw):
    make = FAMILIES[family][0]
    return make(center_init=torch.zeros(B, d, dtype=torch.float64), stdev_init=1.0, objective_sense="min", popsize=popsize, **kw)


# ------------------------------------------------------------------------------------------------ the tables
def _check_row(lad, t: int, ref):
    lam = lad.popsizes[t]
    assert int(lad.counts[t]) == lam == ref.popsize
    assert torch.equal(lad.weights[t, :lam], ref.weights) and not lad.weights[t, lam:].any(), t
    assert lad.consts[t].tolist() == [float(v) for v in _consts(ref)], t
    assert int(lad.decompose_C_freq[t]) == ref.decompose_C_freq and int(lad.history[t]) == lad.history_lengths[t]


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("limit", [True, False])
def test_every_row_up_to_640_is_the_default_of_its_popsize(family, limit):
    d = 7
    state = _state(family, d=d, popsize=10, limit_C_decomposition=limit)
    lad = bipop_ladder(state, 2, 640)
    ipop = ipop_ladder(state, 2, 640)
    K = lad.n_large
    assert lad.popsizes[:K] == ipop.popsizes == (10, 20, 40, 80, 160, 320, 640) and ipop.n_large is None
    assert lad.popsizes[K:] == tuple(range(10, 321)) and lad.weights.shape == (K + 311, 640)
    assert lad.history_lengths == tuple(10 + math.ceil(30 * d / lam) for lam in lad.popsizes)
    assert torch.equal(lad.weights[:K], ipop.weights) and torch.equal(lad.consts[:K], ipop.consts) and len(lad.hyperparameters) == K
    for t, lam in enumerate(lad.popsizes):
        _check_row(lad, t, _state(family, d=d, popsize=lam, limit_C_decomposition=limit).hyperparameters)


def test_rows_at_8192():
    state = _state("cmaes", d=10, popsize=10)
    lad = bipop_ladder(state, 2, 8192)
    K = lad.n_large
    assert lad.popsizes[:K] == (10, 20, 40, 80, 160, 320, 640, 1280, 2560, 5120, 8192)
    assert lad.popsizes[K:] == tuple(range(10, 4097)) and lad.weights.shape == (K + 4087, 8192)
    for lam in (10, 11, 997, 2048, 4095, 4096):
        _check_row(lad, K + lam - 10, _state("cmaes", d=10, popsize=lam).hyperparameters)
    _check_row(lad, K - 1, _state("cmaes", d=10, popsize=8192).hyperparameters)


def test_one_rung_ladder_has_one_small_tier():
    lad = bipop_ladder(_state("cmaes"), 2, 10)
    assert lad.popsizes == (10, 10) and lad.n_large == 1


# ------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("kw", [dict(), dict(popsize_multiplier=2), dict(max_popsize=40), dict(popsize_multiplier=1.0, max_popsize=40),
                                dict(popsize_multiplier=2, max_popsize=9), dict(popsize_multiplier=1.05, max_popsize=40)])
def test_bipop_arguments_are_validated(kw):
    with pytest.raises(ValueError):
        restarts(_state("cmaes"), lb=-1.0, ub=1.0, bipop=True, **kw)


@pytest.mark.parametrize("ratio", ["c_sigma_ratio", "c_mu_ratio", "c_m"])
def test_bipop_rejects_non_default_learning_rates(ratio):
    with pytest.raises(ValueError, match="default learning rates"):
        restarts(_state("sepcmaes", **{ratio: 0.7}), lb=-1.0, ub=1.0, popsize_multiplier=2, max_popsize=40, bipop=True)


def test_fields_are_none_without_bipop():
    for kw in (dict(), dict(popsize_multiplier=2, max_popsize=40)):
        rs = restarts(_state("cmaes"), lb=-1.0, ub=1.0, **kw)
        assert all(getattr(rs, k) is None for k in BIPOP_FIELDS)
        assert rs.ladder is None or rs.ladder.n_large is None


def test_fresh_bipop_state():
    state = _state("sepcmaes", B=3)
    state = state._replace(sigma=torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64))
    rs = restarts(state, lb=-1.0, ub=1.0, popsize_multiplier=2, max_popsize=40, bipop=True)
    assert rs.search.popsize == 40 and rs.ladder.n_large == 3 and rs.ladder.popsizes == (10, 20, 40) + tuple(range(10, 21))
    for k in ("regime", "large_tier", "tier"):
        assert getattr(rs, k).dtype == torch.int32 and not getattr(rs, k).any()
    for k in ("large_evaluations", "small_evaluations", "last_large_evaluations", "num_evaluations"):
        assert getattr(rs, k).dtype == torch.int64 and not getattr(rs, k).any()
    assert torch.equal(rs.run_stdev, state.sigma) and torch.equal(rs.stdev_init, state.sigma) and rs.popsize.tolist() == [10] * 3


# ------------------------------------------------------------------------------------------------ the restart stage
def _torch_stage(c: dict, seed: int, multiplier: float):
    """The torch restart stage on a constructed case in float64; returns (its outputs, the centre u and the policy u it drew)."""
    t = lambda k: torch.tensor(c[k], dtype=torch.float64)  # noqa: E731
    B, D = c["B"], c["D"]
    C = t("c_diag") if c["separable"] else torch.diag_embed(t("c_diag"))
    A = t("r_diag") if c["separable"] else torch.diag_embed(t("r_diag"))
    st = dict(m=t("m"), sigma=t("sigma"), p_sigma=t("p_sigma"), p_c=t("p_c"), C=C, A=A, s=t("sigma")[:, None] * t("r_diag") if c["separable"] else None)
    ints = lambda k, dt=torch.int64: torch.tensor(c[k], dtype=dt)  # noqa: E731
    r = dict(history=t("history"), best_x=t("best_x"), best_f=t("best_f"), num_restarts=ints("num_restarts"), tier=ints("tier", torch.int32),
             num_evaluations=ints("num_evaluations"), regime=ints("regime", torch.int32), large_tier=ints("large_tier", torch.int32),
             large_evaluations=ints("large_evaluations"), small_evaluations=ints("small_evaluations"),
             last_large_evaluations=ints("last_large_evaluations"), run_stdev=t("run_stdev"))
    ladder = bipop_ladder(sepcmaes(center_init=torch.zeros(D, dtype=torch.float64), stdev_init=1.0, objective_sense="min", popsize=6), multiplier, 16)
    assert list(ladder.popsizes) == c["sizes"] and ladder.n_large == c["K"] and list(ladder.history_lengths) == c["hist"]
    torch.manual_seed(seed)
    u = torch.rand(B, D, dtype=torch.float64).numpy()
    u_policy = torch.rand(B, 2, dtype=torch.float64).numpy()
    torch.manual_seed(seed)
    out = _restart_torch(c["thresholds"], c["separable"], c["maximize"], t("f"), t("X"), torch.tensor(c["gen"]), st, r, t("sigma_def"), t("lb"),
                         t("ub"), ladder=ladder)
    return out, u, u_policy


@pytest.mark.parametrize("separable", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
@pytest.mark.parametrize("multiplier", [2.0, 1.5])
def test_torch_stage_against_oracle(separable, maximize, multiplier):
    c = BO.constructed_bipop_items(separable, maximize, multiplier=multiplier)
    (st, r, gen, flags), u, u_policy = _torch_stage(c, 5, multiplier)
    exp = BO.expected(c, u, u_policy, float32=False)
    for b, e in enumerate(exp):
        assert int(flags[b]) == e["flags"], (b, int(flags[b]), e["flags"])
        np.testing.assert_array_equal(r["history"][b].numpy(), e["history"])
        np.testing.assert_array_equal(r["best_x"][b].numpy(), e["best_x"])
        assert float(r["best_f"][b]) == e["best_f"]
        for k in ("tier", "num_evaluations", "regime", "large_tier", "large_evaluations", "small_evaluations", "last_large_evaluations"):
            assert int(r[k][b]) == e[k], (b, k, int(r[k][b]), e[k])
        assert float(r["run_stdev"][b]) == e["run_stdev"], b
        assert int(gen[b]) == e["gen"] and int(r["num_restarts"][b]) == e["num_restarts"]
        if e["reset"]:
            np.testing.assert_array_equal(st["m"][b].numpy(), e["centre"])
            assert float(st["sigma"][b]) == e["run_stdev"]
            if separable:
                assert (st["s"][b] == e["run_stdev"]).all() and (st["C"][b] == 1).all()
        else:
            np.testing.assert_array_equal(st["m"][b].numpy(), c["m"][b])
    _assert_branches(c, exp, multiplier)


def _assert_branches(c: dict, exp: list, multiplier: float):
    """Every branch of the policy fires where the construction puts it."""
    for b, bit in BO.RO.DESIGNED.items():
        assert exp[b]["flags"] & bit and exp[b + 10]["flags"] & bit, (b, bit)
    K, sdef = c["K"], c["sigma_def"]
    assert exp[0]["flags"] == 0 and exp[9]["flags"] == 0 and exp[18]["flags"] == 0
    assert (exp[1]["regime"], exp[1]["tier"], exp[1]["run_stdev"]) == (1, 1, sdef[1])  # the first restart: 0 vs 0 goes large
    assert exp[7]["regime"] == 1 and exp[7]["large_evaluations"] <= exp[7]["small_evaluations"] == 112
    if multiplier == 2.0:
        assert exp[7]["large_evaluations"] == 112  # a tie goes large
    assert exp[6]["regime"] == 1 and exp[6]["tier"] == 1  # large after a small run, one rung up
    for b in (3, 4, 5, 12, 13, 14, 15, 16):  # small chosen
        assert exp[b]["regime"] == 2 and exp[b]["tier"] == K + exp[b]["small_popsize"] - 6 and exp[b]["run_stdev"] <= sdef[b]
    assert exp[4]["small_popsize"] == 6  # lambda_l / 2 = lambda_0 (multiplier 2) or below it (1.5): clamped to lambda_0
    assert exp[5]["flags"] == 32 | 128 and exp[8]["flags"] == 128  # bit 7 with max_generations, and alone at 2 g n = n_last
    assert exp[10]["flags"] == 4 and exp[13]["flags"] & 2  # tol_x_up / tol_x only because of run_stdev
    assert exp[15]["last_large_evaluations"] == 60 * c["sizes"][2]  # a finished large run sets n_last
    if multiplier == 2.0:
        assert exp[2]["tier"] == exp[17]["tier"] == K - 1 == exp[2]["large_tier"]  # the top rung stays
    else:
        assert c["sizes"][1] / 2 < 6 and exp[4]["tier"] == K


def test_budget_bit_boundaries():
    assert BO.budget_bit(2, 5, 6, 60) == 128 and BO.budget_bit(2, 5, 6, 61) == 0 and BO.budget_bit(1, 50, 6, 0) == 0
    assert BO.small_popsize(10, 20, 0.999) == 10 and BO.small_popsize(10, 15, 0.9) == 10 and BO.small_popsize(10, 640, 0.0) == 10
    assert BO.small_popsize(10, 640, 0.99999994) == 319  # floor(10 * 32^(u^2)) just below 320


# ------------------------------------------------------------------------------------------------ a hand-worked schedule
@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
def test_hand_worked_schedule(family):
    """lambda_0 = 10, m = 2 (ladder 10, 20, 40, 80), every run stopped at 5 generations: the first run (50 evaluations in no
    budget); large at 20 (n_L = 100, n_last = 100); small runs at lambda_s = 10 (floor(20 / 2) = lambda_0), each stopped by
    max_generations and bit 7 together (2 * 5 * 10 = 100 = n_last), until n_S = 100 >= n_L; then large at 40 (n_L = 300,
    n_last = 200), and small runs from rung 2 until n_S reaches 300 again."""
    make, ask, _ = FAMILIES[family]
    torch.manual_seed(3)
    state = make(center_init=torch.randn(3, 4, dtype=torch.float64), stdev_init=torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64), objective_sense="min",
                 popsize=10)
    rs = restarts(state, lb=-1.0, ub=1.0, tol_fun=None, tol_x=None, tol_x_up=None, max_condition=None, max_generations=5, popsize_multiplier=2,
                  max_popsize=80, bipop=True)
    seq = []
    for _ in range(20):
        values = ask(rs.search)
        rs = restarts_tell(rs, values, (values * values).sum(-1))
        seq.append(tuple(tuple(getattr(rs, k).tolist()) for k in ("regime", "tier", "large_evaluations", "small_evaluations", "stop_flags")))
    K = 4
    one = lambda regime, tier, n_l, n_s, flags: (regime, tier, n_l, n_s, flags)  # noqa: E731
    expect = ([one(0, 0, 0, 0, 0)] * 4 + [one(1, 1, 0, 0, 32)]  # the first run, then its restart: large at rung 1
              + [one(1, 1, 20 * g, 0, 0) for g in range(1, 5)] + [one(2, K, 100, 0, 32)]  # large at 20; then small at 10
              + [one(2, K, 100, 10 * g, 0) for g in range(1, 5)] + [one(2, K, 100, 50, 32 | 128)]  # a small run, n_S = 50 < 100
              + [one(2, K, 100, 50 + 10 * g, 0) for g in range(1, 5)] + [one(1, 2, 100, 100, 32 | 128)])  # n_S = 100 >= n_L: large at 40
    for g, (row, e) in enumerate(zip(seq, expect)):
        assert row == tuple((v,) * 3 for v in e), (g, row, e)
    assert (rs.large_tier == 2).all() and (rs.last_large_evaluations == 100).all() and (rs.num_evaluations == 50 + 100 + 50 + 50).all()
    assert torch.equal(rs.run_stdev, state.sigma) and torch.equal(rs.search.sigma, state.sigma)
    for _ in range(5):  # the large run at 40: n_L = 300, n_last = 200, then a small run from rung 2 (lambda_s in [10, 20])
        values = ask(rs.search)
        rs = restarts_tell(rs, values, (values * values).sum(-1))
    assert (rs.large_evaluations == 300).all() and (rs.last_large_evaluations == 200).all() and (rs.regime == 2).all()
    lam = rs.popsize
    assert ((lam >= 10) & (lam <= 20)).all() and torch.equal(rs.tier.long(), K + lam - 10)
    assert ((rs.run_stdev <= state.sigma) & (rs.run_stdev > state.sigma / 100)).all() and torch.equal(rs.search.sigma, rs.run_stdev)


# ------------------------------------------------------------------------------------------------ whole runs, float64
def _one_item(state, b: int, generation: int, hp):
    fields = {k: getattr(state, k)[b:b + 1] for k in state._fields if isinstance(getattr(state, k), torch.Tensor)}
    return state._replace(generation=generation, hyperparameters=hp, **fields)


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 7])
def test_torch_run_against_one_item_searches(family, d):
    """Every tell of a run with forced restarts (max_generations 3): an item at tier t equals a one-item search of popsize
    lambda_t told the item's first lambda_t rows (IPOP's tolerances: relative 1e-14, absolute 1e-15), and a restarted item equals
    a fresh search of its next popsize started at its new run_stdev.  Pad rows hold NaN."""
    make, ask, tell = FAMILIES[family]
    torch.manual_seed(12)
    B = 6
    state = make(center_init=torch.randn(B, d, dtype=torch.float64), stdev_init=torch.linspace(0.5, 1.5, B, dtype=torch.float64),
                 objective_sense="min", popsize=4, limit_C_decomposition=False if family == "cmaes" else True)
    rs = restarts(state, lb=-3.0, ub=3.0, max_generations=3, popsize_multiplier=2, max_popsize=20, bipop=True)
    lad, sigma0 = rs.ladder, state.sigma.clone()
    assert lad.popsizes == (4, 8, 16, 20) + tuple(range(4, 11))
    seen = set()
    for g in range(30):
        values = ask(rs.search)
        evals = (values * values).sum(-1)
        lam = rs.popsize
        pad = torch.arange(20) >= lam[:, None]
        values = torch.where(pad[:, :, None], math.nan, values)
        evals = torch.where(pad, math.inf if g % 2 else math.nan, evals)
        nxt = restarts_tell(rs, values, evals)
        for b in range(B):
            t = int(rs.tier[b])
            seen.add((int(rs.regime[b]), t))
            n = lad.popsizes[t]
            assert int(nxt.num_evaluations[b]) == int(rs.num_evaluations[b]) + n
            if nxt.stop_flags[b]:
                assert int(nxt.item_generation[b]) == 0 and float(nxt.search.sigma[b]) == float(nxt.run_stdev[b])
                fresh = make(center_init=nxt.search.center[b:b + 1], stdev_init=nxt.run_stdev[b:b + 1], objective_sense="min")
                for name in FIELDS:
                    assert torch.equal(getattr(nxt.search, name)[b:b + 1], getattr(fresh, name)), (g, b, name)
                if int(nxt.regime[b]) == 1:
                    assert float(nxt.run_stdev[b]) == float(sigma0[b])
            else:
                assert int(nxt.tier[b]) == t and torch.equal(nxt.run_stdev[b], rs.run_stdev[b])
                hp = _state(family, B=1, d=d, popsize=n, limit_C_decomposition=family != "cmaes").hyperparameters
                one = tell(_one_item(rs.search, b, int(rs.item_generation[b]), hp), values[b:b + 1, :n], evals[b:b + 1, :n])
                for name in FIELDS + (("s",) if family == "sepcmaes" else ()):
                    torch.testing.assert_close(getattr(nxt.search, name)[b:b + 1], getattr(one, name), rtol=1e-14, atol=1e-15, msg=f"{g} {b} {name}")
        rs = nxt
    assert {r for r, _ in seen} == {0, 1, 2} and any(t >= lad.n_large + 1 for _, t in seen)  # a small run above lambda_0


# ------------------------------------------------------------------------------------------------ C ABI, no device work
@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


RESTART_BASE = dict(separable=0, f=P, X=P, sx=40, ldx=5, m_draw=None, s_draw=None, draw_seed=0, items=0, N=8, D=5, maximize=0, steps=P, m=P, sigma=P,
                    p_sigma=P, p_c=P, C=P, A=P, s=None, history=P, H=40, best_x=P, best_f=P, num_restarts=P, stop_flags=P, sigma0=P, lb=P, ub=P,
                    sb=5, th="th", seed=1, tier=P, counts=P, hist=P, K=5, evals=P, regime=P, large_tier=P, n_l=P, n_s=P, n_last=P, run_stdev=P,
                    n_large=3, lam0=4)
RESTART_CASES = [
    ({}, 0),
    (dict(separable=1, s=P), 0),
    (dict(separable=1, s=P, X=None, m_draw=P, s_draw=P), 0),
    (dict(f=None), NULLPTR),
    (dict(th=None), NULLPTR),
    (dict(X=None), NULLPTR),
    (dict(tier=None), NULLPTR),
    (dict(evals=None), NULLPTR),
    (dict(regime=None), NULLPTR),
    (dict(large_tier=None), NULLPTR),
    (dict(n_l=None), NULLPTR),
    (dict(n_s=None), NULLPTR),
    (dict(n_last=None), NULLPTR),
    (dict(run_stdev=None), NULLPTR),
    (dict(run_stdev=None, items=-1, n_large=0), NULLPTR),  # null pointers come before sizes
    (dict(items=-1), BADSIZE),
    (dict(N=0), BADSIZE),
    (dict(K=0), BADSIZE),
    (dict(n_large=0), BADSIZE),
    (dict(n_large=5), BADSIZE),  # no small tier
    (dict(n_large=4), 0),
    (dict(lam0=0), BADSIZE),
    (dict(K=0, n_large=0), BADSIZE),
]


@pytest.mark.parametrize("changes,code", RESTART_CASES)
def test_restart_bipop_codes(lib, changes, code):
    a = dict(RESTART_BASE, **changes)
    th = None if a["th"] is None else ops._host_floats([math.nan] * 6, 6)
    before = lib.evok_launch_count()
    rc = lib.evok_cma_restart_batched_bipop(
        a["separable"], a["f"], a["X"], a["sx"], a["ldx"], a["m_draw"], a["s_draw"], a["draw_seed"], a["items"], a["N"], a["D"], a["maximize"], a["steps"],
        a["m"], a["sigma"], a["p_sigma"], a["p_c"], a["C"], a["A"], a["s"], a["history"], a["H"], a["best_x"], a["best_f"], a["num_restarts"],
        a["stop_flags"], a["sigma0"], a["lb"], a["ub"], a["sb"], th, a["seed"], a["tier"], a["counts"], a["hist"], a["K"], a["evals"], a["regime"],
        a["large_tier"], a["n_l"], a["n_s"], a["n_last"], a["run_stdev"], a["n_large"], a["lam0"], None)
    assert lib.evok_launch_count() == before
    assert rc == code
