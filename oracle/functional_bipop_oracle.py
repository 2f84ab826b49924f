"""BIPOP restarts of the functional CMA-ES families (funcrestarts with bipop=True, evok_cma_restart_batched_bipop), restated per
item in float64 numpy on top of the IPOP and restart oracles: the budgets of the two regimes, the small-run budget stop (bit 7),
tol_x and tol_x_up against the step size the run started with, and the choice of the next run at a restart.

Tiers 0..K-1 are IPOP's ladder lambda_0 .. lambda_{K-1}; tier K + (lambda - lambda_0) is a small run of population size lambda.
At a restart the next run is large when n_L <= n_S: rung l <- min(l + 1, K - 1) at the default step size sigma_def.  Otherwise
small: lambda_s = max(lambda_0, floor(lambda_0 exp(u1^2 log(0.5 lambda_l / lambda_0)))) and run_stdev = sigma_def 10^(-2 u2) (rounded
to float32 on the kernels), with u1, u2 = uniform24 of words x, y of Philox4x32-10 at counter (0, 1, 0xFF000000, b) under the
stage's reset key (`bipop_uniforms`).
"""

from __future__ import annotations

import math

import numpy as np

from . import functional_ipop_oracle as IO
from . import functional_restart_oracle as RO
from .es_oracle import philox4x32_10
from .noise_oracle import _key, uniform24

SMALL_BUDGET = 128  # stop bit 7
REGIME_FIRST, REGIME_LARGE, REGIME_SMALL = 0, 1, 2


def tables(lam0: int, multiplier: float, max_popsize: int) -> tuple:
    """(population size of every tier, K): the ladder, then lambda_0 .. max(lambda_0, max_popsize // 2)."""
    sizes = IO.ladder(lam0, multiplier, max_popsize)
    return sizes + list(range(lam0, max(lam0, max_popsize // 2) + 1)), len(sizes)


def bipop_uniforms(seed: int, B: int) -> np.ndarray:
    """[B, 2] float64: u1, u2 of every item's small-run draw on the kernels."""
    b = np.arange(B, dtype=np.uint64)
    zero = np.zeros_like(b)
    words = philox4x32_10(zero, zero + np.uint64(1), np.full_like(b, RO.RESET_TAG), b & np.uint64(0xFFFFFFFF), *_key(seed, 0))
    return np.stack([uniform24(words[0]), uniform24(words[1])], axis=-1).astype(np.float64)


def small_popsize_raw(lam0: int, lam_l: int, u1: float) -> float:
    """lambda_0 exp(u1^2 log(0.5 lambda_l / lambda_0)) in float64, before the floor and the clamp."""
    return lam0 * math.exp(u1 * u1 * math.log(0.5 * lam_l / lam0))


def small_popsize(lam0: int, lam_l: int, u1: float) -> int:
    return max(lam0, int(math.floor(small_popsize_raw(lam0, lam_l, u1))))


def small_stdev(sigma_def: float, u2: float, float32: bool) -> float:
    v = float(sigma_def) * 10.0 ** (-2.0 * float(u2))
    return float(np.float32(v)) if float32 else v


def next_run(*, sizes, K: int, regime: int, large_tier: int, tier: int, gen: int, n: int, large_evaluations: int, small_evaluations: int,
             last_large_evaluations: int, sigma_def: float, u, float32: bool) -> dict:
    """The policy fields of a restarting item whose run (regime, n rows per generation, gen generations) was just accounted."""
    last = gen * n if regime == REGIME_LARGE else last_large_evaluations
    if large_evaluations <= small_evaluations:
        lt = min(large_tier + 1, K - 1)
        return dict(regime=REGIME_LARGE, large_tier=lt, tier=lt, run_stdev=float(sigma_def), last_large_evaluations=last, small_popsize=None)
    lam = small_popsize(sizes[0], sizes[large_tier], float(u[0]))
    return dict(regime=REGIME_SMALL, large_tier=large_tier, tier=min(K + lam - sizes[0], len(sizes) - 1),
                run_stdev=small_stdev(sigma_def, u[1], float32), last_large_evaluations=last, small_popsize=lam)


def account(regime: int, n: int, large_evaluations: int, small_evaluations: int) -> tuple:
    """(n_L, n_S) after a tell of n rows in `regime` (the first run counts in neither)."""
    return large_evaluations + (n if regime == REGIME_LARGE else 0), small_evaluations + (n if regime == REGIME_SMALL else 0)


def budget_bit(regime: int, gen: int, n: int, last_large_evaluations: int) -> int:
    """Bit 7: a small run whose evaluations gen * n reach half the latest large run's (2 gen n >= n_last)."""
    return SMALL_BUDGET if regime == REGIME_SMALL and 2 * gen * n >= last_large_evaluations else 0


def restart_item_bipop(*, sizes, K: int, hist, tier: int, num_evaluations: int, regime: int, large_tier: int, large_evaluations: int,
                       small_evaluations: int, last_large_evaluations: int, run_stdev: float, sigma_def: float, u_policy, f, x_rows, history,
                       gen: int, lb, ub, u, float32: bool, **kw) -> dict:
    """One item of a BIPOP stage: RO.restart_item on its first sizes[tier] rows and hist[tier] slots with tol_x / tol_x_up against
    run_stdev, the budgets, bit 7, then (on a restart) the reset with the next run's step size and the next run's policy fields."""
    n, H = sizes[tier], hist[tier]
    ring = np.array(history, np.float64)
    out = RO.restart_item(f=np.asarray(f)[:n], x_rows=np.asarray(x_rows)[:n], history=ring[:H], gen=gen, sigma0=run_stdev, lb=lb, ub=ub, u=u,
                          float32=float32, **kw)
    n_l, n_s = account(regime, n, large_evaluations, small_evaluations)
    flags = out["flags"] | budget_bit(regime, gen, n, last_large_evaluations)
    res = dict(out, flags=flags, reset=flags != 0, num_evaluations=num_evaluations + n, large_evaluations=n_l, small_evaluations=n_s,
               regime=regime, large_tier=large_tier, tier=tier, run_stdev=float(run_stdev), last_large_evaluations=last_large_evaluations,
               small_popsize=None)
    if flags and not out["reset"]:  # bit 7 alone: the reset restart_item did not do
        res.update(centre=RO.centre(lb, ub, u, float32), gen=0, num_restarts=out["num_restarts"] + 1)
    if flags:
        ring[:] = math.nan
        res.update(next_run(sizes=sizes, K=K, regime=regime, large_tier=large_tier, tier=tier, gen=gen, n=n, large_evaluations=n_l,
                            small_evaluations=n_s, last_large_evaluations=last_large_evaluations, sigma_def=sigma_def, u=u_policy, float32=float32))
    else:
        ring[:H] = out["history"]
    res["history"] = ring
    return res


# item -> (regime, large_tier, small popsize or None, n_L, n_S, n_last, gen or None, run_stdev factor or None); see constructed_bipop_items
_POLICY = {
    0: (0, 0, None, 0, 0, 0, None, None),          # nothing fires: the first run goes on
    1: (0, 0, None, 0, 0, 0, None, None),          # tol_x in the first run: the first restart, 0 vs 0 goes large, rung 1
    2: (1, 2, None, 500, 600, 0, None, None),      # tol_x_up in a top-rung large run, n_L + 16 <= n_S: large again, the top rung stays
    3: (1, 2, None, 400, 100, 0, None, None),      # max_condition in a large run, n_L > n_S: small, lambda_s drawn in [6, 8]
    4: (1, 1, None, 300, 0, 0, None, None),        # min_fitness_stdev at rung 1: small with floor(lambda_1 / 2) = lambda_0: lambda_s = 6
    5: (2, 0, 7, 100, 50, 100, 60, None),          # max_generations and bit 7 together in a small run: small again
    6: (2, 0, 7, 100, 200, 100, None, None),       # non-finite in a small run, n_L <= n_S: large, rung 0 -> 1
    7: (1, 1, None, 100, 112, 0, None, None),      # tol_fun at rung 1, n_L = n_S after the tell: large (ties go large)
    8: (2, 1, 6, 120, 30, 60, 5, None),            # bit 7 alone, at the boundary 2 g n = n_last, with NaN / inf fitnesses
    9: (2, 1, 8, 120, 30, 81, 5, None),            # no finite fitness, 2 g n = 80 < n_last: nothing fires
    10: (2, 2, 7, 100, 10, 1000, None, 1e-5),      # tol_x_up only because the run started at a small step size
    11: (0, 0, None, 0, 0, 0, None, None),         # tol_x in the first run
    12: (2, 2, 8, 50, 40, 1000, None, None),       # tol_x_up in a small run: small again from rung 2
    13: (2, 2, 6, 100, 10, 1000, None, 1e13),      # max_condition, and tol_x only because of the large run_stdev
    14: (1, 0, None, 0, 0, 0, None, None),         # min_fitness_stdev in a large run at rung 0: n_L = 6 > 0, small from lambda_0
    15: (1, 2, None, 30, 10, 0, None, None),       # max_generations in a top-rung large run: n_last = 60 * 16
    16: (2, 1, 6, 100, 30, 1000, None, None),      # non-finite in a small run
    17: (2, 2, 8, 300, 400, 1000, None, None),     # tol_fun in a small run, n_L <= n_S: large, the top rung stays
    18: (1, 1, None, 10, 0, 0, None, None),        # NaN / inf fitnesses in a large run: nothing fires
    19: (0, 0, None, 0, 0, 0, None, None),         # no finite fitness in the first run: nothing fires
}


def constructed_bipop_items(separable: bool, maximize: bool, D: int = 5, seed: int = 0, multiplier: float = 2.0) -> dict:
    """Twenty items: RO.constructed_items twice (items b and b + 10 carry the designed criterion of item b), on the tables of
    (lambda_0 = 6, `multiplier`, max_popsize 16), with the policy states of _POLICY: every branch of the next-run choice, the
    top rung staying, lambda_s clamped to lambda_0 (rung 1 of multiplier 2, where floor(lambda_1 / 2) = lambda_0, and with a
    multiplier < 2, where lambda_1 / 2 < lambda_0), bit 7 alone and with another criterion, tol_x and tol_x_up firing only
    because of run_stdev.  Pad rows of values and fitnesses hold NaN, +-inf and huge values."""
    sizes, K = tables(6, multiplier, 16)
    hist = IO.history_lengths(D, sizes)
    N = sizes[K - 1]
    a = RO.constructed_items(separable, maximize, D=D, N=N, seed=seed)
    b = RO.constructed_items(separable, maximize, D=D, N=N, seed=seed + 1)
    c = {k: (np.concatenate([a[k], b[k]]) if isinstance(a[k], np.ndarray) else a[k]) for k in a}
    B = c["B"] = 2 * a["B"]
    rng = np.random.default_rng(seed + 2)
    c["history"] = np.asarray(rng.normal(size=(B, hist[0])), np.float32).astype(np.float64)
    for t in (7, 17):
        c["history"][t] = 2.0
        c["gen"][t] = hist[0] + 3
    c["num_evaluations"] = rng.integers(0, 1000, B)
    c["sigma_def"] = c["sigma0"]
    fields = ("regime", "large_tier", "tier", "large_evaluations", "small_evaluations", "last_large_evaluations")
    for k in fields:
        c[k] = np.zeros(B, np.int64)
    c["run_stdev"] = c["sigma_def"].copy()
    for item, (reg, lt, lam, n_l, n_s, n_last, gen, factor) in _POLICY.items():
        lt = min(lt, K - 1)
        c["regime"][item], c["large_tier"][item] = reg, lt
        c["tier"][item] = K + lam - sizes[0] if reg == REGIME_SMALL else (lt if reg == REGIME_LARGE else 0)
        c["large_evaluations"][item], c["small_evaluations"][item], c["last_large_evaluations"][item] = n_l, n_s, n_last
        if gen is not None:
            c["gen"][item] = gen
        if reg == REGIME_SMALL:
            c["run_stdev"][item] = float(np.float32(c["sigma_def"][item] * (factor if factor is not None else 0.1)))
    for t in range(B):
        n = sizes[c["tier"][t]]
        for i in range(n, N):
            c["f"][t, i] = IO.PAD[i % len(IO.PAD)]
            c["X"][t, i] = IO.PAD[(i + t) % len(IO.PAD)]
    c.update(sizes=sizes, K=K, hist=hist, H=hist[0])
    return c


def expected(c: dict, u: np.ndarray, u_policy: np.ndarray, float32: bool) -> list:
    """restart_item_bipop for every item of a `constructed_bipop_items` case."""
    rows = c.get("rows", c["X"])
    return [restart_item_bipop(sizes=c["sizes"], K=c["K"], hist=c["hist"], tier=int(c["tier"][b]), num_evaluations=int(c["num_evaluations"][b]),
                               regime=int(c["regime"][b]), large_tier=int(c["large_tier"][b]), large_evaluations=int(c["large_evaluations"][b]),
                               small_evaluations=int(c["small_evaluations"][b]), last_large_evaluations=int(c["last_large_evaluations"][b]),
                               run_stdev=float(c["run_stdev"][b]), sigma_def=float(c["sigma_def"][b]), u_policy=u_policy[b], f=c["f"][b],
                               x_rows=rows[b], history=c["history"][b], gen=int(c["gen"][b]), sigma=float(c["sigma"][b]), m=c["m"][b],
                               p_sigma=c["p_sigma"][b], p_c=c["p_c"][b], c_diag=c["c_diag"][b], r_diag=c["r_diag"][b], separable=c["separable"],
                               best_x=c["best_x"][b], best_f=c["best_f"][b], num_restarts=int(c["num_restarts"][b]), lb=c["lb"][b], ub=c["ub"][b],
                               thresholds=c["thresholds"], maximize=c["maximize"], u=u[b], float32=float32)
            for b in range(c["B"])]


def replay(flags_per_generation, u_per_generation, *, sizes, K: int, sigma_def, float32: bool, gen0: int = 0) -> dict:
    """Every item's policy from its stop flags: flags [G, B] (the stop_flags after each tell), u [G, B, 2] (u1, u2 of each tell's
    draw).  Starting from a fresh BIPOP state (first run at tier 0, item generation gen0), derives after every tell the regime,
    large_tier, tier, the three budgets, run_stdev, num_evaluations and the item generation ([G, B] each), and `budget`: the bit 7
    the policy predicts for each tell, to be compared with the flags' own."""
    flags = np.asarray(flags_per_generation, np.int64)
    G, B = flags.shape
    sigma_def = np.broadcast_to(np.asarray(sigma_def, np.float64), (B,))
    names = ("regime", "large_tier", "tier", "large_evaluations", "small_evaluations", "last_large_evaluations", "num_evaluations", "gen", "budget")
    out = {k: np.zeros((G, B), np.int64) for k in names}
    out["run_stdev"] = np.zeros((G, B))
    for b in range(B):
        s = dict(regime=0, large_tier=0, tier=0, large_evaluations=0, small_evaluations=0, last_large_evaluations=0, num_evaluations=0, gen=gen0)
        stdev = float(np.float32(sigma_def[b])) if float32 else float(sigma_def[b])
        for g in range(G):
            n = sizes[s["tier"]]
            s["gen"] += 1
            s["num_evaluations"] += n
            s["large_evaluations"], s["small_evaluations"] = account(s["regime"], n, s["large_evaluations"], s["small_evaluations"])
            out["budget"][g, b] = budget_bit(s["regime"], s["gen"], n, s["last_large_evaluations"])
            if flags[g, b]:
                nxt = next_run(sizes=sizes, K=K, regime=s["regime"], large_tier=s["large_tier"], tier=s["tier"], gen=s["gen"], n=n,
                               large_evaluations=s["large_evaluations"], small_evaluations=s["small_evaluations"],
                               last_large_evaluations=s["last_large_evaluations"], sigma_def=sigma_def[b], u=u_per_generation[g][b], float32=float32)
                stdev = nxt["run_stdev"]
                s.update(regime=nxt["regime"], large_tier=nxt["large_tier"], tier=nxt["tier"], last_large_evaluations=nxt["last_large_evaluations"],
                         gen=0)
            for k in names[:-1]:
                out[k][g, b] = s[k]
            out["run_stdev"][g, b] = stdev
    return out
