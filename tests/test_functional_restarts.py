"""Restarts of the functional CMA-ES families without a GPU: the torch restart stage against the float64 oracle on constructed
states where each criterion fires on one item and not on the others, whole float64 runs on the torch path (per-item counters,
forced restarts), argument validation, and the return codes of the new C entry points on calls that launch nothing."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_tell, restarts, restarts_tell, sepcmaes, sepcmaes_ask, sepcmaes_tell
from evotorch_b200.algorithms.functional.funcrestarts import _restart_torch, history_length
from oracle import functional_restart_oracle as RO

NULLPTR, BADSIZE = -1, -2
P = 64  # any non-null pointer: the argument checks never dereference it


def _torch_stage(c: dict, seed: int):
    """The torch restart stage on a constructed case in float64; returns (its outputs, the u it drew)."""
    t = lambda k: torch.tensor(c[k], dtype=torch.float64)  # noqa: E731
    B, D = c["B"], c["D"]
    C = t("c_diag") if c["separable"] else torch.diag_embed(t("c_diag"))
    A = t("r_diag") if c["separable"] else torch.diag_embed(t("r_diag"))
    st = dict(m=t("m"), sigma=t("sigma"), p_sigma=t("p_sigma"), p_c=t("p_c"), C=C, A=A, s=t("sigma")[:, None] * t("r_diag") if c["separable"] else None)
    r = dict(history=t("history"), best_x=t("best_x"), best_f=t("best_f"), num_restarts=torch.tensor(c["num_restarts"]))
    torch.manual_seed(seed)
    u = torch.rand(B, D, dtype=torch.float64).numpy()
    torch.manual_seed(seed)
    out = _restart_torch(c["thresholds"], c["separable"], c["maximize"], t("f"), t("X"), torch.tensor(c["gen"]), st, r, t("sigma0"), t("lb"), t("ub"))
    return out, u


@pytest.mark.parametrize("separable", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
def test_torch_stage_against_oracle(separable, maximize):
    c = RO.constructed_items(separable, maximize)
    (st, r, gen, flags), u = _torch_stage(c, seed=7)
    exp = RO.expected(c, u, float32=False)
    D = c["D"]
    for b, e in enumerate(exp):
        assert int(flags[b]) == e["flags"], (b, int(flags[b]), e["flags"])
        np.testing.assert_array_equal(r["best_x"][b].numpy(), e["best_x"])
        assert float(r["best_f"][b]) == e["best_f"]
        np.testing.assert_array_equal(r["history"][b].numpy(), e["history"])
        assert int(gen[b]) == e["gen"] and int(r["num_restarts"][b]) == e["num_restarts"]
        if e["reset"]:
            np.testing.assert_array_equal(st["m"][b].numpy(), e["centre"])
            assert float(st["sigma"][b]) == c["sigma0"][b]
            assert not st["p_sigma"][b].any() and not st["p_c"][b].any()
            one = torch.ones(D, dtype=torch.float64) if separable else torch.eye(D, dtype=torch.float64)
            assert torch.equal(st["C"][b], one) and torch.equal(st["A"][b], one)
            if separable:
                assert torch.equal(st["s"][b], torch.full((D,), c["sigma0"][b], dtype=torch.float64))
        else:
            np.testing.assert_array_equal(st["m"][b].numpy(), c["m"][b])
            assert float(st["sigma"][b]) == c["sigma"][b]
    for b, bit in RO.DESIGNED.items():
        assert exp[b]["flags"] & bit, (b, bit)
    assert exp[0]["flags"] == 0 and exp[8]["flags"] == 0
    assert exp[0]["best_x"].tolist() == c["X"][0, 2].tolist()  # the lower row of a tie
    assert exp[8]["best_f"] == c["best_f"][8] and math.isnan(exp[9]["history"][4])


@pytest.mark.parametrize("separable", [False, True])
def test_each_threshold_turns_its_criterion_off(separable):
    c = RO.constructed_items(separable, False)
    for k, name in enumerate(ops.RESTART_CRITERIA):
        th = list(c["thresholds"])
        th[k] = None
        (_, _, _, flags), u = _torch_stage(dict(c, thresholds=tuple(th)), seed=1)
        assert not (flags & (1 << k)).any(), name
        assert [e["flags"] for e in RO.expected(dict(c, thresholds=tuple(th)), u, False)] == flags.tolist()


def _one_item(state, b: int, generation: int):
    """Item b of a state (batch shape (B,)) as a one-item state with its own generation counter."""
    fields = {k: getattr(state, k)[b:b + 1] for k in state._fields if isinstance(getattr(state, k), torch.Tensor)}
    return state._replace(generation=generation, **fields)


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 7])
def test_torch_run_against_one_item_tells(family, d):
    """Every tell with forced restarts: a restarted item equals a fresh search at its new centre, every other item the family's
    tell of its one-item state at its own counter."""
    make, ask, tell = (cmaes, cmaes_ask, cmaes_tell) if family == "cmaes" else (sepcmaes, sepcmaes_ask, sepcmaes_tell)
    torch.manual_seed(3)
    B = 5
    state = make(center_init=torch.randn(B, d, dtype=torch.float64), stdev_init=torch.linspace(0.5, 1.5, B, dtype=torch.float64),
                 objective_sense="min")
    rs = restarts(state, lb=-3.0, ub=torch.linspace(1.0, 3.0, d, dtype=torch.float64), max_generations=torch.tensor(4))
    sigma0 = state.sigma.clone()
    for g in range(12):
        values = ask(rs.search)
        evals = (values * values).sum(-1)
        evals[g % B, 1] = math.nan
        nxt = restarts_tell(rs, values, evals)
        assert nxt.search.generation == rs.search.generation + 1
        for b in range(B):
            if nxt.stop_flags[b]:
                fresh = make(center_init=nxt.search.center[b:b + 1], stdev_init=sigma0[b:b + 1], objective_sense="min")
                assert int(nxt.item_generation[b]) == 0 and int(nxt.stop_flags[b]) == 32
                for k in ("center", "sigma", "C", "A", "p_sigma", "p_c") + (("s",) if family == "sepcmaes" else ()):
                    assert torch.equal(getattr(nxt.search, k)[b:b + 1], getattr(fresh, k)), (g, b, k)
            else:
                one = tell(_one_item(rs.search, b, int(rs.item_generation[b])), values[b:b + 1], evals[b:b + 1])
                assert int(nxt.item_generation[b]) == int(rs.item_generation[b]) + 1
                for k in ("center", "sigma", "C", "A", "p_sigma", "p_c") + (("s",) if family == "sepcmaes" else ()):
                    torch.testing.assert_close(getattr(nxt.search, k)[b:b + 1], getattr(one, k), rtol=1e-14, atol=1e-300, msg=f"{g} {b} {k}")
        rs = nxt
    assert (rs.num_restarts >= 2).all()
    assert torch.isfinite(rs.best_evals).all() and not torch.isnan(rs.best_values).any()


def test_restarts_tell_leaves_its_input_unchanged():
    torch.manual_seed(0)
    rs = restarts(cmaes(center_init=torch.randn(3, 4, dtype=torch.float64), stdev_init=1.0, objective_sense="max"), lb=-1.0, ub=1.0,
                  max_generations=1)
    before = [t.clone() if isinstance(t, torch.Tensor) else t for t in rs]
    values = cmaes_ask(rs.search)
    nxt = restarts_tell(rs, values, values.sum(-1))
    assert (nxt.stop_flags == 32).all() and (nxt.num_restarts == 1).all()
    for a, b in zip(before, rs):
        if isinstance(a, torch.Tensor):
            assert torch.equal(a, b) or (a.isnan() == b.isnan()).all()
    assert (rs.best_evals == -math.inf).all() and (nxt.best_evals > -math.inf).all()


def test_restart_state_fields():
    state = sepcmaes(center_init=torch.zeros(2, 3, 6, dtype=torch.float64), stdev_init=0.3, objective_sense="min", popsize=8)
    state = state._replace(generation=4)
    rs = restarts(state, lb=torch.full((6,), -2.0), ub=torch.full((3, 6), 2.0), tol_fun=None, max_condition=1e10)
    H = history_length(6, 8)
    assert H == 10 + math.ceil(30 * 6 / 8)
    assert rs.history.shape == (2, 3, H) and rs.history.isnan().all()
    assert rs.item_generation.dtype == torch.int64 and (rs.item_generation == 4).all()
    assert rs.stop_flags.dtype == torch.int32 and rs.num_restarts.dtype == torch.int64
    assert rs.lb.shape == rs.ub.shape == (2, 3, 6) and (rs.stdev_init == 0.3).all()
    assert rs.thresholds == (None, 1e-12, 1e4, 1e10, None, None)
    assert (rs.best_evals == math.inf).all() and rs.best_values.isnan().all()


@pytest.mark.parametrize("lb,ub", [(1.0, 1.0), (2.0, 1.0), (-math.inf, 1.0), (0.0, math.nan), (torch.zeros(4), torch.ones(5)),
                                   (torch.zeros(2, 3), 1.0)])
def test_bounds_are_validated(lb, ub):
    state = cmaes(center_init=torch.zeros(3, 5, dtype=torch.float64), stdev_init=1.0, objective_sense="min")
    with pytest.raises(ValueError):
        restarts(state, lb=lb, ub=ub)


def test_arguments_are_validated():
    state = cmaes(center_init=torch.zeros(5, dtype=torch.float64), stdev_init=1.0, objective_sense="min")
    with pytest.raises(TypeError):
        restarts(state._asdict(), lb=-1.0, ub=1.0)
    with pytest.raises(ValueError):
        restarts(state, lb=-1.0, ub=1.0, tol_x=torch.ones(2))
    rs = restarts(state, lb=-1.0, ub=1.0)
    with pytest.raises(ValueError):
        restarts_tell(rs, torch.zeros(state.popsize + 1, 5), torch.zeros(state.popsize + 1))


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


RESTART_BASE = dict(separable=0, f=P, X=P, sx=40, ldx=5, m_draw=None, s_draw=None, draw_seed=0, items=0, N=8, D=5, maximize=0, steps=P, m=P, sigma=P,
                    p_sigma=P, p_c=P, C=P, A=P, s=None, history=P, H=40, best_x=P, best_f=P, num_restarts=P, stop_flags=P, sigma0=P, lb=P, ub=P,
                    sb=5, th="th", seed=1)
RESTART_CASES = [
    ({}, 0),
    (dict(separable=1, s=P), 0),
    (dict(separable=1, s=P, X=None, m_draw=P, s_draw=P), 0),
    (dict(sb=0), 0),
    (dict(f=None), NULLPTR),
    (dict(steps=None), NULLPTR),
    (dict(history=None), NULLPTR),
    (dict(th=None), NULLPTR),
    (dict(X=None), NULLPTR),  # the full family needs its population
    (dict(separable=1), NULLPTR),  # s
    (dict(separable=1, s=P, X=None, m_draw=P), NULLPTR),
    (dict(f=None, items=-1), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(N=0), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(H=0), BADSIZE),
    (dict(ldx=4), BADSIZE),
    (dict(sx=-1), BADSIZE),
    (dict(sb=3), BADSIZE),
    (dict(separable=1, s=P, X=None, m_draw=P, s_draw=P, ldx=0, sx=-1), 0),  # no X: its strides are not read
]


def restart_call(lib, a):
    th = None if a["th"] is None else ops._host_floats([math.nan] * 6, 6)
    return lib.evok_cma_restart_batched(a["separable"], a["f"], a["X"], a["sx"], a["ldx"], a["m_draw"], a["s_draw"], a["draw_seed"], a["items"], a["N"],
                                        a["D"], a["maximize"], a["steps"], a["m"], a["sigma"], a["p_sigma"], a["p_c"], a["C"], a["A"], a["s"],
                                        a["history"], a["H"], a["best_x"], a["best_f"], a["num_restarts"], a["stop_flags"], a["sigma0"], a["lb"], a["ub"],
                                        a["sb"], th, a["seed"], None)


@pytest.mark.parametrize("changes,code", RESTART_CASES)
def test_restart_codes(lib, changes, code):
    assert _no_launch(lib, lambda: restart_call(lib, dict(RESTART_BASE, **changes))) == code


CONSTS = ops._host_floats([0.5] * 10, 10)


@pytest.mark.parametrize("changes,code", [({}, 0), (dict(steps=None), NULLPTR), (dict(m=None), NULLPTR), (dict(items=-1), BADSIZE), (dict(D=0), BADSIZE)])
def test_vector_update_steps_codes(lib, changes, code):
    a = dict(dict(items=0, D=4, m=P, steps=P), **changes)
    assert _no_launch(lib, lambda: lib.evok_cmaes_vector_update_batched_steps(P, P, a["items"], a["D"], a["m"], P, P, P, a["steps"], CONSTS, 0, P,
                                                                              None)) == code


@pytest.mark.parametrize("changes,code", [({}, 0), (dict(steps=None), NULLPTR), (dict(C=None), NULLPTR), (dict(items=-1), BADSIZE), (dict(D=0), BADSIZE),
                                          (dict(freq=0), BADSIZE)])
def test_sepcma_update_steps_codes(lib, changes, code):
    a = dict(dict(items=0, D=4, C=P, steps=P, freq=1), **changes)
    assert _no_launch(lib, lambda: lib.evok_sepcma_update_batched_steps(P, P, P, a["items"], a["D"], P, P, P, P, a["C"], P, P, a["steps"], CONSTS, 0,
                                                                        a["freq"], math.nan, math.nan, None)) == code
