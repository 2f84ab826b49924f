"""IPOP restarts of the functional CMA-ES families without a GPU: the ladder and its validation, the constants of each tier, the
torch restart stage on padded populations against the float64 oracle, whole float64 runs checked item by item against one-item
searches of the item's population size, pad rows that hold NaN / inf / huge values, and the return codes of the tiered C entry
points on calls that launch nothing."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask, cmaes_tell, ipop_ladder, restarts, restarts_tell, sepcmaes, sepcmaes_ask,
                                                 sepcmaes_tell)
from evotorch_b200.algorithms.functional.funcrestarts import _restart_torch
from oracle import functional_ipop_oracle as IO

NULLPTR, BADSIZE = -1, -2
P = 64  # any non-null pointer: the argument checks never dereference it
FAMILIES = {"cmaes": (cmaes, cmaes_ask, cmaes_tell), "sepcmaes": (sepcmaes, sepcmaes_ask, sepcmaes_tell)}
FIELDS = ("center", "sigma", "C", "A", "p_sigma", "p_c")


def _state(family: str, B: int = 4, d: int = 3, popsize: int = 10, **kw):
    make = FAMILIES[family][0]
    return make(center_init=torch.zeros(B, d, dtype=torch.float64), stdev_init=1.0, objective_sense="min", popsize=popsize, **kw)


# ------------------------------------------------------------------------------------------------ the ladder
def test_ladder_doubles_to_the_cap():
    rs = restarts(_state("cmaes"), lb=-1.0, ub=1.0, popsize_multiplier=2, max_popsize=640)
    assert rs.ladder.popsizes == (10, 20, 40, 80, 160, 320, 640) == tuple(IO.ladder(10, 2, 640))
    assert rs.search.popsize == 640 and rs.history.shape[-1] == rs.ladder.history_lengths[0] == 10 + math.ceil(90 / 10)
    assert rs.ladder.history_lengths == tuple(10 + math.ceil(30 * 3 / lam) for lam in rs.ladder.popsizes)
    assert rs.tier.dtype == torch.int32 and not rs.tier.any() and rs.num_evaluations.dtype == torch.int64 and not rs.num_evaluations.any()
    assert rs.popsize.tolist() == [10] * 4
    assert ipop_ladder(_state("sepcmaes"), 2, 100).popsizes == (10, 20, 40, 80, 100)  # a cap that is not a rung ends the ladder
    assert ipop_ladder(_state("cmaes"), 1.5, 10).popsizes == (10,)
    assert ipop_ladder(_state("cmaes"), 2.5, 70).popsizes == (10, 25, 62, 70)  # int(2.5 * 25) = 62


@pytest.mark.parametrize("kw", [dict(popsize_multiplier=1.0, max_popsize=40), dict(popsize_multiplier=0.5, max_popsize=40),
                                dict(popsize_multiplier=2, max_popsize=9), dict(popsize_multiplier=1.05, max_popsize=40),
                                dict(popsize_multiplier=2), dict(max_popsize=40), dict(popsize_multiplier=torch.ones(2) * 2, max_popsize=40)])
def test_ladder_arguments_are_validated(kw):
    with pytest.raises(ValueError):
        restarts(_state("cmaes"), lb=-1.0, ub=1.0, **kw)


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("ratio", ["c_sigma_ratio", "c_1_ratio", "c_mu_ratio", "damp_sigma_ratio", "c_c_ratio", "c_m"])
def test_non_default_learning_rates_are_rejected(family, ratio):
    with pytest.raises(ValueError, match="default learning rates"):
        restarts(_state(family, **{ratio: 0.7}), lb=-1.0, ub=1.0, popsize_multiplier=2, max_popsize=40)


def test_plain_restart_state_has_no_ipop_fields():
    rs = restarts(_state("cmaes"), lb=-1.0, ub=1.0)
    assert rs.tier is None and rs.num_evaluations is None and rs.ladder is None
    assert rs.popsize.tolist() == [10] * 4 and rs.search.popsize == 10


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("limit", [True, False])
@pytest.mark.parametrize("active", [True, False])
def test_tier_constants_are_those_of_the_popsize(family, limit, active):
    state = _state(family, d=7, popsize=6, limit_C_decomposition=limit, active=active)
    lad = ipop_ladder(state, 2, 200)
    assert lad.popsizes == (6, 12, 24, 48, 96, 192, 200)
    for k, lam in enumerate(lad.popsizes):
        ref = _state(family, d=7, popsize=lam, limit_C_decomposition=limit, active=active).hyperparameters
        hp = lad.hyperparameters[k]
        for name, a, b in zip(hp._fields, hp, ref):
            assert torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b, (k, name)
        assert torch.equal(lad.weights[k, :lam], ref.weights) and not lad.weights[k, lam:].any()
        assert lad.consts[k].tolist() == [float(v) for v in (ref.c_m, ref.c_sigma, ref.damp_sigma, ref.c_c, ref.c_1, ref.c_mu, ref.variance_discount_sigma,
                                                              ref.variance_discount_c, ref.unbiased_expectation, ref.weights_sum)]
        assert int(lad.decompose_C_freq[k]) == ref.decompose_C_freq and int(lad.counts[k]) == lam
        assert int(lad.history[k]) == 10 + math.ceil(30 * 7 / lam)


# ------------------------------------------------------------------------------------------------ the restart stage
def _torch_stage(c: dict, seed: int):
    """The torch restart stage on a constructed tiered case in float64; returns (its outputs, the u it drew)."""
    t = lambda k: torch.tensor(c[k], dtype=torch.float64)  # noqa: E731
    B, D = c["B"], c["D"]
    C = t("c_diag") if c["separable"] else torch.diag_embed(t("c_diag"))
    A = t("r_diag") if c["separable"] else torch.diag_embed(t("r_diag"))
    st = dict(m=t("m"), sigma=t("sigma"), p_sigma=t("p_sigma"), p_c=t("p_c"), C=C, A=A, s=t("sigma")[:, None] * t("r_diag") if c["separable"] else None)
    r = dict(history=t("history"), best_x=t("best_x"), best_f=t("best_f"), num_restarts=torch.tensor(c["num_restarts"]),
             tier=torch.tensor(c["tier"], dtype=torch.int32), num_evaluations=torch.tensor(c["num_evaluations"]))
    ladder = ipop_ladder(sepcmaes(center_init=torch.zeros(D, dtype=torch.float64), stdev_init=1.0, objective_sense="min", popsize=6), 2, 16)
    assert list(ladder.popsizes) == c["sizes"] and list(ladder.history_lengths) == c["hist"]
    torch.manual_seed(seed)
    u = torch.rand(B, D, dtype=torch.float64).numpy()
    torch.manual_seed(seed)
    out = _restart_torch(c["thresholds"], c["separable"], c["maximize"], t("f"), t("X"), torch.tensor(c["gen"]), st, r, t("sigma0"), t("lb"), t("ub"),
                         ladder=ladder)
    return out, u


@pytest.mark.parametrize("separable", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
def test_torch_stage_against_oracle(separable, maximize):
    c = IO.constructed_tiered_items(separable, maximize)
    (st, r, gen, flags), u = _torch_stage(c, seed=5)
    exp = IO.expected(c, u, float32=False)
    for b, e in enumerate(exp):
        assert int(flags[b]) == e["flags"], (b, int(flags[b]), e["flags"])
        np.testing.assert_array_equal(r["history"][b].numpy(), e["history"])
        np.testing.assert_array_equal(r["best_x"][b].numpy(), e["best_x"])
        assert float(r["best_f"][b]) == e["best_f"]
        assert int(r["tier"][b]) == e["tier"] and int(r["num_evaluations"][b]) == e["num_evaluations"], b
        assert int(gen[b]) == e["gen"] and int(r["num_restarts"][b]) == e["num_restarts"]
        if e["reset"]:
            np.testing.assert_array_equal(st["m"][b].numpy(), e["centre"])
    for b, bit in IO.RO.DESIGNED.items():
        assert exp[b]["flags"] & bit, (b, bit)
    assert exp[0]["flags"] == 0 and exp[8]["flags"] == 0
    assert {int(c["tier"][b]) for b in range(c["B"]) if exp[b]["reset"]} == {0, 1, 2}  # every tier restarts somewhere
    assert exp[2]["tier"] == 2 and exp[1]["tier"] == 2  # the top tier stays; tier 1 moves up


def test_oracle_ranks_only_the_first_rows():
    w = np.array([0.5, 0.3, 0.2, -0.1])
    f = [3.0, math.nan, 1.0, 2.0, -math.inf, math.nan]
    assert IO.assigned_weights(f, 4, w, False).tolist() == [0.2, -0.1, 0.5, 0.3, 0.0, 0.0]
    assert IO.assigned_weights(f, 4, w, True).tolist() == [0.3, 0.5, -0.1, 0.2, 0.0, 0.0]


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("maximize", [False, True])
def test_torch_ranking_against_oracle(family, maximize):
    from evotorch_b200.algorithms.functional.funccmaes import _assigned_weights

    lad = ipop_ladder(_state(family, popsize=6), 2, 16)
    rng = np.random.default_rng(2)
    f = rng.normal(size=(9, 16)).round(1)
    f[:, ::5] = math.nan
    f[3, 1] = math.inf
    tier = torch.arange(9) % 3
    real = torch.arange(16) < lad.counts.long()[tier][:, None]
    got = _assigned_weights(torch.tensor(f), maximize, lad.weights[tier], real)
    for b in range(9):
        k = int(tier[b])
        assert got[b].tolist() == IO.assigned_weights(f[b], lad.popsizes[k], lad.weights[k].numpy(), maximize).tolist(), b


# ------------------------------------------------------------------------------------------------ whole runs, float64
def _one_item(state, b: int, generation: int, hp):
    fields = {k: getattr(state, k)[b:b + 1] for k in state._fields if isinstance(getattr(state, k), torch.Tensor)}
    return state._replace(generation=generation, hyperparameters=hp, **fields)


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 7])
def test_torch_run_against_one_item_searches(family, d):
    """Every tell of a run with forced restarts (max_generations 3): an item at tier k equals a one-item search of popsize
    lambda_k told the item's first lambda_k rows and evals at the item's own counter (float64, relative tolerance 1e-14 and
    absolute 1e-15: the covariance product sums over all max_popsize rows, the zero ones too, so its partial sums may be grouped
    differently); a restarted item equals a fresh search of the next popsize.  Pad rows hold NaN."""
    make, ask, tell = FAMILIES[family]
    torch.manual_seed(11)
    B = 5
    state = make(center_init=torch.randn(B, d, dtype=torch.float64), stdev_init=torch.linspace(0.5, 1.5, B, dtype=torch.float64),
                 objective_sense="min", popsize=4, limit_C_decomposition=False if family == "cmaes" else True)
    rs = restarts(state, lb=-3.0, ub=3.0, max_generations=3, popsize_multiplier=2, max_popsize=20)
    assert rs.ladder.popsizes == (4, 8, 16, 20)
    lad, sigma0 = rs.ladder, state.sigma.clone()
    seen = set()
    for g in range(16):
        values = ask(rs.search)
        evals = (values * values).sum(-1)
        lam = rs.popsize
        pad = torch.arange(20) >= lam[:, None]
        values = torch.where(pad[:, :, None], math.nan, values)
        evals = torch.where(pad, math.inf if g % 2 else math.nan, evals)
        evals[g % B, 1] = math.nan
        nxt = restarts_tell(rs, values, evals)
        for b in range(B):
            k = int(rs.tier[b])
            seen.add(k)
            n = lad.popsizes[k]
            assert int(nxt.num_evaluations[b]) == int(rs.num_evaluations[b]) + n
            if nxt.stop_flags[b]:
                assert int(nxt.tier[b]) == min(k + 1, 3) and int(nxt.item_generation[b]) == 0
                fresh = make(center_init=nxt.search.center[b:b + 1], stdev_init=sigma0[b:b + 1], objective_sense="min")
                for name in FIELDS:
                    assert torch.equal(getattr(nxt.search, name)[b:b + 1], getattr(fresh, name)), (g, b, name)
            else:
                assert int(nxt.tier[b]) == k
                one = tell(_one_item(rs.search, b, int(rs.item_generation[b]), lad.hyperparameters[k]), values[b:b + 1, :n], evals[b:b + 1, :n])
                for name in FIELDS + (("s",) if family == "sepcmaes" else ()):
                    torch.testing.assert_close(getattr(nxt.search, name)[b:b + 1], getattr(one, name), rtol=1e-14, atol=1e-15, msg=f"{g} {b} {name}")
            assert torch.isfinite(nxt.best_evals[b])
        rs = nxt
    assert seen == {0, 1, 2, 3}


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("maximize", [False, True])
def test_pad_rows_reach_nothing(family, maximize):
    """NaN, +-inf and huge values in the pad rows of values and evals leave every state tensor as finite pad rows do."""
    make, ask, _ = FAMILIES[family]
    torch.manual_seed(4)
    B, d = 6, 4
    state = make(center_init=torch.randn(B, d, dtype=torch.float64), stdev_init=0.7, objective_sense="max" if maximize else "min", popsize=5)
    rs = restarts(state, lb=-2.0, ub=2.0, max_generations=2, min_fitness_stdev=1e-3, popsize_multiplier=2, max_popsize=25)
    for g in range(7):
        values = ask(rs.search)
        evals = -(values * values).sum(-1)
        pad = torch.arange(25) >= rs.popsize[:, None]
        outs = []
        for fill_x, fill_f in ((0.0, 0.0), (math.nan, math.nan), (math.inf, -math.inf), (-1e300, 1e300), (1e300, -math.inf)):
            torch.manual_seed(100 + g)
            outs.append(restarts_tell(rs, torch.where(pad[:, :, None], fill_x, values), torch.where(pad, fill_f, evals)))
        for o in outs[1:]:
            for a, b in zip(outs[0], o):
                if isinstance(a, torch.Tensor):
                    assert torch.equal(a, b) or torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())
                elif isinstance(a, tuple):
                    for x, y in zip(a, b):
                        assert x is y or torch.equal(x, y) or (isinstance(x, torch.Tensor) and torch.equal(x.nan_to_num(), y.nan_to_num()))
        rs = outs[0]
    assert (rs.tier > 0).any()


def test_restarts_tell_leaves_its_input_unchanged():
    torch.manual_seed(0)
    rs = restarts(sepcmaes(center_init=torch.randn(3, 4, dtype=torch.float64), stdev_init=1.0, objective_sense="max", popsize=6), lb=-1.0, ub=1.0,
                  max_generations=1, popsize_multiplier=3, max_popsize=50)
    before = [t.clone() for t in (rs.tier, rs.num_evaluations)]
    values = sepcmaes_ask(rs.search)
    nxt = restarts_tell(rs, values, values.sum(-1))
    assert torch.equal(before[0], rs.tier) and torch.equal(before[1], rs.num_evaluations)
    assert (nxt.tier == 1).all() and (nxt.num_evaluations == 6).all() and nxt.popsize.tolist() == [18] * 3


# ------------------------------------------------------------------------------------------------ C ABI, no device work
@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def _no_launch(lib, call):
    before = lib.evok_launch_count()
    rc = call()
    assert lib.evok_launch_count() == before
    return rc


@pytest.mark.parametrize("changes,code", [({}, 0), (dict(N=0), 0), (dict(keys=None), NULLPTR), (dict(tables=None), NULLPTR), (dict(tier=None), NULLPTR),
                                          (dict(counts=None), NULLPTR), (dict(out=None), NULLPTR), (dict(N=-1), BADSIZE), (dict(N=8193), BADSIZE),
                                          (dict(N=8192), 0), (dict(items=-1), BADSIZE), (dict(tier=None, N=8193), NULLPTR)])
def test_rank_tiered_codes(lib, changes, code):
    a = dict(dict(keys=P, N=16, items=0, tables=P, tier=P, counts=P, out=P), **changes)
    assert _no_launch(lib, lambda: lib.evok_rank_table_batched_tiered(a["keys"], a["N"], a["items"], 0, a["tables"], a["tier"], a["counts"], a["out"],
                                                                      None)) == code


@pytest.mark.parametrize("changes,code", [({}, 0), (dict(tier=None), NULLPTR), (dict(counts=None), NULLPTR), (dict(Z=None), NULLPTR),
                                          (dict(tier=None, N=0), NULLPTR), (dict(items=-1), BADSIZE), (dict(N=0), BADSIZE), (dict(ldz=2), BADSIZE)])
def test_row_weights_tiered_codes(lib, changes, code):
    a = dict(dict(Z=P, items=0, N=8, ldz=3, tier=P, counts=P), **changes)
    assert _no_launch(lib, lambda: lib.evok_cmaes_row_weights_batched_tiered(P, a["Z"], 24, a["ldz"], a["items"], a["N"], 3, 1, a["tier"], a["counts"],
                                                                             P, P, None)) == code


@pytest.mark.parametrize("changes,code", [({}, 0), (dict(steps=None), NULLPTR), (dict(tier=None), NULLPTR), (dict(consts=None), NULLPTR),
                                          (dict(m=None), NULLPTR), (dict(items=-1), BADSIZE), (dict(D=0), BADSIZE)])
def test_vector_update_tiered_codes(lib, changes, code):
    a = dict(dict(items=0, D=4, m=P, steps=P, tier=P, consts=P), **changes)
    assert _no_launch(lib, lambda: lib.evok_cmaes_vector_update_batched_tiered(P, P, a["items"], a["D"], a["m"], P, P, P, a["steps"], a["tier"],
                                                                               a["consts"], 0, P, None)) == code


@pytest.mark.parametrize("changes,code", [({}, 0), (dict(steps=None), NULLPTR), (dict(tier=None), NULLPTR), (dict(consts=None), NULLPTR),
                                          (dict(freq=None), NULLPTR), (dict(C=None), NULLPTR), (dict(items=-1), BADSIZE), (dict(D=0), BADSIZE)])
def test_sepcma_update_tiered_codes(lib, changes, code):
    a = dict(dict(items=0, D=4, C=P, steps=P, tier=P, consts=P, freq=P), **changes)
    assert _no_launch(lib, lambda: lib.evok_sepcma_update_batched_tiered(P, P, P, a["items"], a["D"], P, P, P, P, a["C"], P, P, a["steps"], a["tier"],
                                                                         a["consts"], a["freq"], 0, math.nan, math.nan, None)) == code


RESTART_BASE = dict(separable=0, f=P, X=P, sx=40, ldx=5, m_draw=None, s_draw=None, draw_seed=0, items=0, N=8, D=5, maximize=0, steps=P, m=P, sigma=P,
                    p_sigma=P, p_c=P, C=P, A=P, s=None, history=P, H=40, best_x=P, best_f=P, num_restarts=P, stop_flags=P, sigma0=P, lb=P, ub=P,
                    sb=5, th="th", seed=1, tier=P, counts=P, hist=P, K=3, evals=P)
RESTART_CASES = [
    ({}, 0),
    (dict(separable=1, s=P), 0),
    (dict(separable=1, s=P, X=None, m_draw=P, s_draw=P), 0),
    (dict(f=None), NULLPTR),
    (dict(th=None), NULLPTR),
    (dict(X=None), NULLPTR),
    (dict(tier=None), NULLPTR),
    (dict(counts=None), NULLPTR),
    (dict(hist=None), NULLPTR),
    (dict(evals=None), NULLPTR),
    (dict(evals=None, items=-1, K=0), NULLPTR),  # null pointers come before sizes
    (dict(items=-1), BADSIZE),
    (dict(N=0), BADSIZE),
    (dict(H=0), BADSIZE),
    (dict(sb=3), BADSIZE),
    (dict(K=0), BADSIZE),
    (dict(K=1), 0),
]


@pytest.mark.parametrize("changes,code", RESTART_CASES)
def test_restart_tiered_codes(lib, changes, code):
    a = dict(RESTART_BASE, **changes)
    th = None if a["th"] is None else ops._host_floats([math.nan] * 6, 6)
    assert _no_launch(lib, lambda: lib.evok_cma_restart_batched_tiered(
        a["separable"], a["f"], a["X"], a["sx"], a["ldx"], a["m_draw"], a["s_draw"], a["draw_seed"], a["items"], a["N"], a["D"], a["maximize"], a["steps"],
        a["m"], a["sigma"], a["p_sigma"], a["p_c"], a["C"], a["A"], a["s"], a["history"], a["H"], a["best_x"], a["best_f"], a["num_restarts"],
        a["stop_flags"], a["sigma0"], a["lb"], a["ub"], a["sb"], th, a["seed"], a["tier"], a["counts"], a["hist"], a["K"], a["evals"], None)) == code
