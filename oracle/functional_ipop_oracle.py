"""IPOP restarts of the functional CMA-ES families on padded populations (funcrestarts with popsize_multiplier, the *_tiered
kernels), restated per item in float64 numpy: the ladder, the ranking of an item's first lambda_k rows, and the tiered restart
stage (the stage of functional_restart_oracle on the first lambda_k values and H_k history slots, then the evaluation count
and the tier advance).  The reset draw is functional_restart_oracle's.
"""

from __future__ import annotations

import math

import numpy as np

from . import functional_restart_oracle as RO


def ladder(lam0: int, multiplier: float, max_popsize: int) -> list:
    """lambda_0 = lam0, lambda_{k+1} = min(int(multiplier * lambda_k), max_popsize) until max_popsize."""
    sizes = [lam0]
    while sizes[-1] < max_popsize:
        sizes.append(min(int(multiplier * sizes[-1]), max_popsize))
    return sizes


def history_lengths(d: int, sizes) -> list:
    return [10 + math.ceil(30 * d / lam) for lam in sizes]


def assigned_weights(f, n: int, weights, maximize: bool) -> np.ndarray:
    """One item: weights[position] for its first n keys (a stable sort under the sense, NaN after every number whatever the sense
    for "min" and before them for "max", as the keys of rank_table_batched order them), 0 for the pad rows."""
    f = np.asarray(f, np.float64)
    N = f.size
    key = np.where(np.isnan(f[:n]), math.inf, f[:n])
    nan_rank = np.isnan(f[:n])
    # sort key: (NaN last ascending / first descending, value), ties by index
    if maximize:
        order = sorted(range(n), key=lambda i: (0 if nan_rank[i] else 1, -key[i], i))
    else:
        order = sorted(range(n), key=lambda i: (1 if nan_rank[i] else 0, key[i], i))
    out = np.zeros(N)
    for p, i in enumerate(order):
        out[i] = float(weights[p])
    return out


def restart_item_tiered(*, tier: int, sizes, hist, num_evaluations: int, f, x_rows, history, **kw) -> dict:
    """RO.restart_item for an item at `tier` of a padded population: the first sizes[tier] values and rows, the first hist[tier]
    slots of its ring (the rest of the ring is kept, or cleared to NaN on a restart); then num_evaluations += sizes[tier] and a
    restarted item moves to min(tier + 1, K - 1)."""
    n, H = sizes[tier], hist[tier]
    ring = np.array(history, np.float64)
    out = RO.restart_item(f=np.asarray(f)[:n], x_rows=np.asarray(x_rows)[:n], history=ring[:H], **kw)
    if out["reset"]:
        ring[:] = math.nan
    else:
        ring[:H] = out["history"]
    out.update(history=ring, num_evaluations=num_evaluations + n, tier=min(tier + 1, len(sizes) - 1) if out["reset"] else tier)
    return out


PAD = (math.nan, math.inf, -math.inf, 3e38, -3e38)


def constructed_tiered_items(separable: bool, maximize: bool, D: int = 5, seed: int = 0) -> dict:
    """The ten items of RO.constructed_items on a padded population of the ladder (6, 12, 16): item b at tier b % 3 (so item 4's
    constant fitnesses, item 7's tol_fun and every other designed criterion fire at some tier, and every tier is present), the
    ring of H_0 slots, and pad rows of values and fitnesses holding NaN, +-inf and huge values."""
    sizes = ladder(6, 2.0, 16)
    hist = history_lengths(D, sizes)
    c = RO.constructed_items(separable, maximize, D=D, N=sizes[-1], seed=seed)
    rng = np.random.default_rng(seed + 1)
    B = c["B"]
    c["history"] = np.asarray(rng.normal(size=(B, hist[0])), np.float32).astype(np.float64)
    c["history"][7] = 2.0
    c["gen"][7] = hist[0] + 3
    c["tier"] = np.arange(B) % len(sizes)
    c["num_evaluations"] = rng.integers(0, 1000, B)
    for b in range(B):
        n = sizes[c["tier"][b]]
        for i in range(n, sizes[-1]):
            c["f"][b, i] = PAD[i % len(PAD)]
            c["X"][b, i] = PAD[(i + b) % len(PAD)]
    c.update(sizes=sizes, hist=hist, H=hist[0])
    return c


def expected(c: dict, u: np.ndarray, float32: bool) -> list:
    """restart_item_tiered for every item of a `constructed_tiered_items` case."""
    rows = c.get("rows", c["X"])
    return [restart_item_tiered(tier=int(c["tier"][b]), sizes=c["sizes"], hist=c["hist"], num_evaluations=int(c["num_evaluations"][b]), f=c["f"][b],
                                x_rows=rows[b], history=c["history"][b], gen=int(c["gen"][b]), sigma=float(c["sigma"][b]), m=c["m"][b],
                                p_sigma=c["p_sigma"][b], p_c=c["p_c"][b], c_diag=c["c_diag"][b], r_diag=c["r_diag"][b], separable=c["separable"],
                                best_x=c["best_x"][b], best_f=c["best_f"][b], num_restarts=int(c["num_restarts"][b]), sigma0=float(c["sigma0"][b]),
                                lb=c["lb"][b], ub=c["ub"][b], thresholds=c["thresholds"], maximize=c["maximize"], u=u[b], float32=float32)
            for b in range(c["B"])]
