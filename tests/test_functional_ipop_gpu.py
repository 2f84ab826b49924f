"""IPOP restarts of the functional CMA-ES families on the H100: every tiered entry against the oracle or the existing entry (bit
for bit), an item at the top tier equal to the non-tiered entry, items independent of the others' tiers, the edges (D, odd and
70 000 items, N = 8192 and 8193), lazy separable runs equal to stored ones with NaN pad rows, no host synchronisation, a launch
count that does not depend on the tiers, and the share of items that reach the optimum of 10-D Rastrigin and Rosenbrock."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import ops
from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask_and_evaluate, ipop_ladder, restarts, restarts_tell, sepcmaes,
                                                 sepcmaes_ask_and_evaluate)
from evotorch_b200.algorithms.functional.funccmaes import _consts
from evotorch_b200.objectives import rastrigin
from oracle import functional_ipop_oracle as IO
from oracle import functional_restart_oracle as RO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _ladder(sizes, N: int, d: int = 5, separable: bool = False):
    """A ladder from sizes[0] that ends at N (float32, on the device)."""
    state = (sepcmaes if separable else cmaes)(center_init=torch.zeros(d, device=DEV), stdev_init=1.0, objective_sense="min", popsize=sizes[0])
    lad = ipop_ladder(state, 2, N)
    return lad


# ------------------------------------------------------------------------------------------------ rank and row weights
@pytest.mark.parametrize("N,B", [(16, 7), (640, 33), (8192, 3), (24, 70_000)])
@pytest.mark.parametrize("maximize", [False, True])
def test_rank_tiered_against_oracle_and_top_tier(N, B, maximize):
    lad = _ladder([max(N // 8, 2)], N)
    K = len(lad.popsizes)
    g = torch.Generator(device=DEV).manual_seed(N + B)
    f = torch.randn(B, N, device=DEV, generator=g).round(decimals=1)
    f[:, ::7] = math.nan
    f[:, 3::11] = math.inf
    tier = (torch.arange(B, device=DEV) % K).to(torch.int32)
    tier[-1] = K - 1  # an item at the top tier, whatever B
    out = ops.rank_table_batched(f, maximize, lad.weights, tier=tier, counts=lad.counts)
    w = lad.weights.cpu().numpy()
    fc, oc = f.cpu().numpy(), out.cpu().numpy()
    for b in list(range(min(B, 2 * K))) + [B - 1]:
        k = int(tier[b])
        np.testing.assert_array_equal(oc[b], IO.assigned_weights(fc[b], lad.popsizes[k], w[k], maximize).astype(np.float32), err_msg=str(b))
    top = tier == K - 1
    ref = ops.rank_table_batched(f[top].contiguous(), maximize, lad.weights[K - 1].contiguous())
    assert torch.equal(_bits(out[top]), _bits(ref))
    if B < 100:  # item independence: one-item calls
        for b in range(B):
            one = ops.rank_table_batched(f[b:b + 1].contiguous(), maximize, lad.weights, tier=tier[b:b + 1].contiguous(), counts=lad.counts)
            assert torch.equal(_bits(one[0]), _bits(out[b]))


def test_rank_tiered_rejects_n_above_8192():
    f = torch.zeros(2, 8193, device=DEV)
    with pytest.raises(ValueError, match="EVOK|size|-2"):
        ops.rank_table_batched(f, False, torch.zeros(1, 8193, device=DEV), tier=torch.zeros(2, dtype=torch.int32, device=DEV),
                               counts=torch.full((1,), 8193, dtype=torch.int32, device=DEV))
    state = cmaes(center_init=torch.zeros(2, device=DEV), stdev_init=1.0, objective_sense="min", popsize=100)
    with pytest.raises(ValueError, match="8192"):
        restarts(state, lb=-1.0, ub=1.0, popsize_multiplier=2, max_popsize=8193)


@pytest.mark.parametrize("d", [1, 3, 33, 130])
@pytest.mark.parametrize("B", [5, 70_000])
def test_row_weights_tiered(d, B):
    if B > 1000 and d > 3:
        pytest.skip("the chunking edge needs one small D")
    lad = _ladder([4], 16)
    K = len(lad.popsizes)
    g = torch.Generator(device=DEV).manual_seed(d)
    Z = torch.randn(B, 16, d, device=DEV, generator=g)
    tier = (torch.arange(B, device=DEV) % K).to(torch.int32)
    real = torch.arange(16, device=DEV) < lad.counts.long()[tier.long()][:, None]
    Z = torch.where(real[:, :, None], Z, math.nan)
    Z[:, :, 0] = torch.where(real, Z[:, :, 0], 0.0)  # a zero row where d = 1: the 0 / 0 the mask must hide
    aw = ops.rank_table_batched(torch.randn(B, 16, device=DEV, generator=g), False, lad.weights, tier=tier, counts=lad.counts)
    w_pos, w_act = torch.full_like(aw, 7.0), torch.full_like(aw, 7.0)
    ops.cmaes_row_weights_batched(aw, Z, True, w_pos, w_act, tier=tier, counts=lad.counts)
    assert not w_pos[~real].any() and not w_act[~real].any()
    rp, ra = torch.empty_like(aw), torch.empty_like(aw)
    ops.cmaes_row_weights_batched(aw, torch.where(real[:, :, None], Z, 1.0), True, rp, ra)
    assert torch.equal(_bits(w_pos[real]), _bits(rp[real])) and torch.equal(_bits(w_act[real]), _bits(ra[real]))


# ------------------------------------------------------------------------------------------------ updates
@pytest.mark.parametrize("d", [1, 3, 33, 130])
def test_vector_and_sepcma_update_tiered_equal_the_untiered_entries(d):
    """Item b with the constants of its tier has the bits of the per-item-counter entry called with that tier's host constants
    (the same kernel code; the constants come from a device table instead of the launch)."""
    B = 9
    for sep in (False, True):
        lad = _ladder([4], 40, d, separable=sep)
        K = len(lad.popsizes)
        g = torch.Generator(device=DEV).manual_seed(d + sep)
        r = lambda *s: torch.randn(*s, device=DEV, generator=g)  # noqa: E731
        tier = (torch.arange(B, device=DEV) % K).to(torch.int32)
        local, shaped, m, ps, pc = (r(B, d) for _ in range(5))
        sigma = r(B).abs() + 0.5
        steps = torch.arange(B, device=DEV, dtype=torch.int64) * 3
        S2, wsum, C = r(B, d).abs(), r(B) * 0.1, r(B, d).abs() + 0.5
        A, s = C.sqrt(), (sigma[:, None] * C.sqrt()).contiguous()
        outs = [t.clone() for t in (m, ps, pc, sigma, steps, C, A, s)]
        k_out = torch.empty(B, 3, device=DEV)
        if sep:
            ops.sepcma_update_batched(local.clone(), S2, wsum, outs[0], outs[1], outs[2], outs[3], outs[5], outs[6], outs[7], lad.consts, False,
                                      steps=outs[4], decompose_C_freq=lad.decompose_C_freq, tier=tier)
        else:
            ops.cmaes_vector_update_batched(local, shaped, outs[0], outs[1], outs[2], outs[3], lad.consts, False, k_out, steps=outs[4], tier=tier)
        for k in range(K):
            sel = (tier == k).nonzero()[:, 0]
            ref = [t[sel].contiguous() for t in (m, ps, pc, sigma, steps, C, A, s)]
            hp = lad.hyperparameters[k]
            if sep:
                ops.sepcma_update_batched(local[sel].contiguous(), S2[sel].contiguous(), wsum[sel].contiguous(), ref[0], ref[1], ref[2], ref[3], ref[5],
                                          ref[6], ref[7], _consts(hp), False, steps=ref[4], decompose_C_freq=hp.decompose_C_freq)
            else:
                kr = torch.empty(len(sel), 3, device=DEV)
                ops.cmaes_vector_update_batched(local[sel].contiguous(), shaped[sel].contiguous(), ref[0], ref[1], ref[2], ref[3], _consts(hp), False, kr,
                                                steps=ref[4])
                assert torch.equal(_bits(k_out[sel]), _bits(kr)), (d, k)
            for a, b in zip(outs, ref):
                assert torch.equal(_bits(a[sel]), _bits(b)), (sep, d, k)


# ------------------------------------------------------------------------------------------------ the restart stage
@pytest.mark.parametrize("separable", [False, True])
@pytest.mark.parametrize("maximize", [False, True])
def test_restart_tiered_against_oracle(separable, maximize):
    c = IO.constructed_tiered_items(separable, maximize)
    seed = 0x2468_ACE0_1357
    t = lambda k: torch.tensor(c[k], dtype=torch.float32, device=DEV).contiguous()  # noqa: E731
    B, D = c["B"], c["D"]
    C = t("c_diag") if separable else torch.diag_embed(t("c_diag")).contiguous()
    A = t("r_diag") if separable else torch.diag_embed(t("r_diag")).contiguous()
    s = (t("sigma")[:, None] * t("r_diag")).contiguous() if separable else None
    o = dict(m=t("m"), sigma=t("sigma"), p_sigma=t("p_sigma"), p_c=t("p_c"), C=C, A=A, s=s, history=t("history"), best_x=t("best_x"),
             best_f=t("best_f"), num_restarts=torch.tensor(c["num_restarts"], device=DEV), steps=torch.tensor(c["gen"], device=DEV),
             flags=torch.full((B,), -1, dtype=torch.int32, device=DEV), tier=torch.tensor(c["tier"], dtype=torch.int32, device=DEV),
             num_evaluations=torch.tensor(c["num_evaluations"], device=DEV))
    lad = _ladder([6], 16, D, separable)
    ops.cma_restart_batched(separable, t("f"), t("X"), maximize, o["steps"], o["m"], o["sigma"], o["p_sigma"], o["p_c"], o["C"], o["A"], o["s"],
                            o["history"], o["best_x"], o["best_f"], o["num_restarts"], o["flags"], t("sigma0"), t("lb"), t("ub"), c["thresholds"],
                            seed=seed, tier=o["tier"], tier_counts=lad.counts, tier_history=lad.history, num_evaluations=o["num_evaluations"])
    o = {k: (v.double() if v.is_floating_point() else v).cpu().numpy() for k, v in o.items() if v is not None}
    exp = IO.expected(c, RO.reset_uniforms(seed, B, D), float32=True)
    for b, e in enumerate(exp):
        assert o["flags"][b] == e["flags"], (b, o["flags"][b], e["flags"])
        np.testing.assert_array_equal(o["best_x"][b], e["best_x"])
        assert o["best_f"][b] == e["best_f"]
        np.testing.assert_array_equal(o["history"][b], e["history"])
        assert o["tier"][b] == e["tier"] and o["num_evaluations"][b] == e["num_evaluations"] and o["steps"][b] == e["gen"]
        if e["reset"]:
            np.testing.assert_array_equal(o["m"][b], e["centre"])
        else:
            np.testing.assert_array_equal(o["m"][b], c["m"][b])
    for b, bit in RO.DESIGNED.items():
        assert o["flags"][b] & bit


# ------------------------------------------------------------------------------------------------ whole runs
def _run(family: str, gens: int, B: int, d: int, lazy: bool = False, tiers=None, pad_nan: bool = False, seed: int = 5):
    torch.manual_seed(seed)
    make = cmaes if family == "cmaes" else sepcmaes
    state = make(center_init=torch.rand(B, d, device=DEV) * 10 - 5, stdev_init=2.0, objective_sense="min", popsize=5)
    rs = restarts(state, lb=-5.0, ub=5.0, max_generations=3, min_fitness_stdev=1e-3, popsize_multiplier=2, max_popsize=40)
    if tiers is not None:
        rs = rs._replace(tier=tiers.clone())
    out = []
    for _ in range(gens):
        if family == "cmaes":
            values, evals = cmaes_ask_and_evaluate(rs.search, objective=rastrigin)
        else:
            values, evals = sepcmaes_ask_and_evaluate(rs.search, objective=rastrigin, lazy=lazy)
        if pad_nan:
            pad = torch.arange(40, device=DEV) >= rs.popsize[:, None]
            values = torch.where(pad[:, :, None], math.nan, values)
            evals = torch.where(pad, math.nan, evals)
        rs = restarts_tell(rs, values, evals)
        out.append(rs)
    return out


def _all(rs) -> list:
    return [_bits(t) for t in list(rs.search) + list(rs) if isinstance(t, torch.Tensor)]


def test_lazy_separable_equals_stored_with_nan_pad_rows():
    stored, lazy = _run("sepcmaes", 14, 9, 40, pad_nan=True), _run("sepcmaes", 14, 9, 40, lazy=True)
    for a, b in zip(stored, lazy):
        for x, y in zip(_all(a), _all(b)):
            assert torch.equal(x, y)
    assert (stored[-1].tier > 0).any() and not stored[-1].best_values.isnan().any()


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
@pytest.mark.parametrize("d", [1, 3, 33, 130])
def test_items_do_not_depend_on_the_others_tiers(family, d):
    """Item 0 at tier 1 in a batch of mixed tiers equals item 0 of a batch where every item is at tier 1, bit for bit."""
    B = 5
    mixed = torch.tensor([1, 0, 3, 2, 3], dtype=torch.int32, device=DEV)
    a = _run(family, 4, B, d, tiers=mixed, seed=7)
    b = _run(family, 4, B, d, tiers=torch.ones(B, dtype=torch.int32, device=DEV), seed=7)
    for ra, rb in zip(a, b):
        for x, y in zip(_all(ra), _all(rb)):
            if x.ndim and x.shape[0] == B:
                assert torch.equal(x[0], y[0])


@pytest.mark.parametrize("family", ["cmaes", "sepcmaes"])
def test_no_host_synchronisation_and_launch_count(family):
    torch.manual_seed(0)
    make = cmaes if family == "cmaes" else sepcmaes
    ask = cmaes_ask_and_evaluate if family == "cmaes" else sepcmaes_ask_and_evaluate
    rs = restarts(make(center_init=torch.randn(33, 9, device=DEV), stdev_init=1.0, objective_sense="min", popsize=6), lb=-3.0, ub=3.0,
                  max_generations=2, min_fitness_stdev=1e-6, popsize_multiplier=2, max_popsize=48)
    pops = []
    for _ in range(5):
        pops.append(ask(rs.search, objective=rastrigin))
        rs = restarts_tell(rs, *pops[-1])
    torch.cuda.synchronize()
    rs = rs._replace(tier=(torch.arange(33, device=DEV) % 4).to(torch.int32))
    counts, tiers = [], []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for values, evals in pops:
            tiers.append(rs.tier.clone())
            before = ops.launch_count()
            rs = restarts_tell(rs, values, evals)
            counts.append(ops.launch_count() - before)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(set(counts)) == 1, counts
    assert len({tuple(t.tolist()) for t in tiers}) > 1  # the mix of tiers changed between the counted generations


# ------------------------------------------------------------------------------------------------ what IPOP buys
def _rosenbrock(x: torch.Tensor) -> torch.Tensor:
    return (100.0 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1.0 - x[..., :-1]) ** 2).sum(-1)


def _share(objective, B: int, gens: int, bound: float, tol_fun: float, popsize: int, ipop: bool) -> tuple:
    torch.manual_seed(123)
    state = cmaes(center_init=torch.rand(B, 10, device=DEV) * 2 * bound - bound, stdev_init=0.3 * bound, objective_sense="min", popsize=popsize)
    kw = dict(popsize_multiplier=2, max_popsize=640) if ipop else {}
    rs = restarts(state, lb=-bound, ub=bound, tol_fun=tol_fun, **kw)
    for _ in range(gens):
        values, evals = cmaes_ask_and_evaluate(rs.search, objective=objective)
        rs = restarts_tell(rs, values, evals)
    n_evals = rs.num_evaluations.double().mean().item() if ipop else float(gens * popsize)
    return (rs.best_evals < 1e-8).float().mean().item(), n_evals, rs.best_evals.isnan().any().item()


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
def test_ipop_reaches_the_optimum(name):
    objective = rastrigin if name == "rastrigin" else _rosenbrock
    bound = 5.12 if name == "rastrigin" else 5.0
    # tol_fun as in the plain restarts test: a flat float32 Rastrigin range is 1e-4
    tol_fun = 1e-4 if name == "rastrigin" else 1e-12
    gens = 2000
    ipop, ipop_evals, nan = _share(objective, 512, gens, bound, tol_fun, 10, True)
    p10, _, _ = _share(objective, 512, gens, bound, tol_fun, 10, False)
    p100, _, _ = _share(objective, 512, gens, bound, tol_fun, 100, False)
    print(f"{name} 10-D, 512 items x {gens} generations, share with f < 1e-8: IPOP from 10 (x2, max 640) {ipop:.3f} at "
          f"{ipop_evals:.0f} evaluations per item; plain restarts popsize 10 {p10:.3f} ({gens * 10} evaluations), popsize 100 {p100:.3f} "
          f"({gens * 100})")
    assert not nan
    # measured on an H100 80GB HBM3: Rastrigin 1.000 (IPOP) / 0.000 (popsize 10) / 0.758 (popsize 100); Rosenbrock 0.932 / 0.930 /
    # 1.000, where tol_fun 1e-12 rarely fires and IPOP stays near popsize 10 (about 20 200 evaluations per item)
    if name == "rastrigin":
        assert ipop > 0.9 and ipop > p10 + 0.5
    else:
        assert ipop > 0.8 and ipop >= p10 - 0.02
