"""BIPOP restarts of the functional CMA-ES families (padded populations) over a batch of B searches (N = lambda_0, D = solution
length), measured against IPOP and plain restarts:
    (a) ms per generation of all B items (ask + fused Rastrigin + restarts_tell) for BIPOP with the ladder N, 2N, ..., 8N and the
        items spread over both regimes (half on the ladder's rungs, half in small runs of sizes N .. 4N), IPOP on the same ladder
        with the items spread over its tiers, and plain restarts at popsize N.  Windows alternate the three; medians.
    (b) the BIPOP restart stage alone against the tiered (IPOP) one on the same padded fitnesses, every item restarting, CUDA
        events, median of 50 launches.
    (c) the share of items whose best ever reaches f < 1e-8 against the mean evaluations per item on 10-D Rastrigin, Rosenbrock
        and the unrotated Lunacek bi-Rastrigin (BBOB f24 without rotation or conditioning, a FusedObjective), for BIPOP and IPOP
        from popsize 10 (x2, max 640) and plain restarts at popsize 10, read at the same evaluation budgets.
The ask draws and evaluates all 8N rows of every item, whatever its regime, which (a) measures.  The card's name and power limit
are read in the same run.

    python scripts/functional_bipop_bench.py [--cmaes 1024x16x32,...] [--sepcmaes 1024x24x1000,...] [--windows 3] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evotorch_b200 import ops  # noqa: E402
from evotorch_b200.algorithms.functional import (SepCMAESState, cmaes, cmaes_ask_and_evaluate, restarts, restarts_tell,  # noqa: E402
                                                 sepcmaes, sepcmaes_ask_and_evaluate)
from evotorch_b200.objectives import rastrigin  # noqa: E402
from scripts.functional_cmaes_bench import card, timed  # noqa: E402
from scripts.functional_ipop_bench import _events  # noqa: E402

DEV = torch.device("cuda")
MULT = 8  # the top of the ladder, in multiples of lambda_0


def lunacek(d: int):
    """The unrotated, unconditioned Lunacek bi-Rastrigin (BBOB f24) as a FusedObjective; optimum 0 at x = 2.5."""
    from evotorch_b200.objectives import FusedObjective

    s = 1.0 - 1.0 / (2.0 * math.sqrt(d + 20.0) - 8.2)
    mu1 = -math.sqrt((2.5 ** 2 - 1.0) / s)
    return FusedObjective("lunacek", sums={"a": "(x - 2.5)**2", "b": f"(x - ({mu1!r}))**2", "c": "cos(6.283185307179586 * (x - 2.5))"},
                          value=f"where(a < D + {s!r} * b, a, D + {s!r} * b) + 10 * (D - c)")


def rosenbrock(x: torch.Tensor) -> torch.Tensor:
    return (100.0 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1.0 - x[..., :-1]) ** 2).sum(-1)


def _spread_bipop(rs, B: int):
    """Half of the items on the ladder's rungs (large runs), half in small runs of every size lambda_0 .. 4 lambda_0."""
    lad = rs.ladder
    K, lam0 = lad.n_large, lad.popsizes[0]
    b = torch.arange(B, device=DEV)
    large = b % 2 == 0
    small_lam = lam0 + (b // 2) % (len(lad.popsizes) - K)
    tier = torch.where(large, (b // 2) % K, K + small_lam - lam0).to(torch.int32)
    return rs._replace(regime=torch.where(large, 1, 2).to(torch.int32), tier=tier, large_tier=torch.where(large, tier, K - 1).to(torch.int32),
                       large_evaluations=torch.full((B,), 10**9, device=DEV), last_large_evaluations=torch.full((B,), 10**9, device=DEV))


def bench_shape(family: str, B: int, n: int, d: int, windows: int) -> dict:
    torch.manual_seed(0)
    make, ask = (cmaes, cmaes_ask_and_evaluate) if family == "cmaes" else (sepcmaes, sepcmaes_ask_and_evaluate)
    centre = torch.rand(B, d, device=DEV) * 4 - 2
    big = n * MULT
    state = lambda popsize: make(center_init=centre, stdev_init=1.0, objective_sense="min", popsize=popsize)  # noqa: E731
    bipop = _spread_bipop(restarts(state(n), lb=-5.12, ub=5.12, popsize_multiplier=2, max_popsize=big, bipop=True), B)
    ipop = restarts(state(n), lb=-5.12, ub=5.12, popsize_multiplier=2, max_popsize=big)
    ipop = ipop._replace(tier=(torch.arange(B, device=DEV) % len(ipop.ladder.popsizes)).to(torch.int32))
    box = {"bipop": bipop, "ipop": ipop, "plain": restarts(state(n), lb=-5.12, ub=5.12)}

    def step(key):
        def run():
            box[key] = restarts_tell(box[key], *ask(box[key].search, objective=rastrigin))
        return run

    fns = {k: step(k) for k in box}
    gens = max(3, min(50, int(2e9 // max(1, B * big * d * (d if family == "cmaes" else 1) * 4))))
    for fn in fns.values():
        fn()
        fn()
    ms = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            ms[k].append(timed(fn, gens))
    out = {"family": family, "B": B, "N": n, "max_popsize": big, "D": d, "gens_per_window": gens,
           "bipop_regimes_at_end": [int((box["bipop"].regime == r).sum()) for r in (0, 1, 2)]}
    for k, label in (("bipop", "bipop_ms"), ("ipop", "ipop_ms"), ("plain", f"plain_popsize_{n}_ms")):
        out[label] = statistics.median(ms[k])
        out[label + "_spread"] = [min(ms[k]), max(ms[k])]
    out.update(stage_ms(_spread_bipop(box["bipop"], B), ask))
    return out


def stage_ms(rs, ask) -> dict:
    """The BIPOP restart stage and the tiered one on the same padded (B, max_popsize) fitnesses, every item restarting."""
    s = rs.search
    sep = isinstance(s, SepCMAESState)
    values, evals = ask(s, objective=rastrigin)
    B, d = s.center.reshape(-1, s.center.shape[-1]).shape
    n = s.popsize
    f, X = evals.reshape(B, n).contiguous(), values.reshape(B, n, d).contiguous()
    lad = rs.ladder
    mat = (B, d) if sep else (B, d, d)
    st = [s.center.reshape(B, d).clone(), s.sigma.reshape(B).clone(), s.p_sigma.reshape(B, d).clone(), s.p_c.reshape(B, d).clone(),
          s.C.reshape(mat).clone(), s.A.reshape(mat).clone(), s.s.reshape(B, d).clone() if sep else None]
    steps = rs.item_generation.reshape(B).clone() + 1
    r = [rs.history.reshape(B, -1).clone(), rs.best_values.reshape(B, d).clone(), rs.best_evals.reshape(B).clone(), rs.num_restarts.reshape(B).clone()]
    flags = torch.empty(B, dtype=torch.int32, device=DEV)
    sig0, lb, ub = rs.stdev_init.reshape(B).contiguous(), rs.lb.reshape(B, d), rs.ub.reshape(B, d)
    args = (sep, f, X, False, steps, *st, *r, flags, sig0, lb, ub, (None,) * 5 + (0.0,))  # max_generations 0: every item restarts
    tier, ne = rs.tier.reshape(B).clone(), rs.num_evaluations.reshape(B).clone()
    pol = {k: getattr(rs, k).reshape(B).clone() for k in ("regime", "large_tier", "large_evaluations", "small_evaluations", "last_large_evaluations",
                                                           "run_stdev")}
    tiers = dict(tier=tier, tier_counts=lad.counts, tier_history=lad.history, num_evaluations=ne)
    return {"restart_bipop_ms": _events(lambda: ops.cma_restart_batched(*args, seed=1, **tiers, **pol, n_large=lad.n_large, popsize0=lad.popsizes[0])),
            "restart_tiered_ms": _events(lambda: ops.cma_restart_batched(*args, seed=1, **tiers))}


def optimum_share(name: str, objective, bound: float, tol_fun: float, B: int, gens: int, every: int) -> dict:
    """Share at the optimum against mean evaluations per item: BIPOP and IPOP checkpoints every `every` generations, then plain
    restarts at popsize 10 read at BIPOP's evaluation budgets."""
    def start(**kw):
        torch.manual_seed(123)
        state = cmaes(center_init=torch.rand(B, 10, device=DEV) * 2 * bound - bound, stdev_init=0.3 * bound, objective_sense="min", popsize=10)
        return restarts(state, lb=-bound, ub=bound, tol_fun=tol_fun, **kw)

    out = {"objective": name, "D": 10, "B": B, "tol_fun": tol_fun}
    for key, kw in (("bipop", dict(bipop=True)), ("ipop", {})):
        rs, curve = start(popsize_multiplier=2, max_popsize=640, **kw), []
        for g in range(1, gens + 1):
            rs = restarts_tell(rs, *cmaes_ask_and_evaluate(rs.search, objective=objective))
            if g % every == 0:
                curve.append({"generations": g, "mean_evaluations": rs.num_evaluations.double().mean().item(),
                              "share": (rs.best_evals < 1e-8).float().mean().item(), "median_best": rs.best_evals.median().item()})
        out[key] = curve
    rs, pts, g = start(), [], 0
    for point in out["bipop"]:
        while (g + 1) * 10 <= point["mean_evaluations"]:
            rs = restarts_tell(rs, *cmaes_ask_and_evaluate(rs.search, objective=objective))
            g += 1
        pts.append({"evaluations": g * 10, "share": (rs.best_evals < 1e-8).float().mean().item(), "median_best": rs.best_evals.median().item()})
    out["plain_popsize_10"] = pts
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cmaes", default="1024x16x32,256x20x128,64x24x512,8x32x2048")
    ap.add_argument("--sepcmaes", default="1024x24x1000,64x200x10000")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--share-items", type=int, default=512)
    ap.add_argument("--share-generations", type=int, default=1000)
    ap.add_argument("--share-every", type=int, default=250)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("functional_bipop_bench.py measures on a CUDA device; none is available")
    out = {"card": card(), "shapes": [], "optimum_share": []}
    for family in ("cmaes", "sepcmaes"):
        for spec in filter(None, getattr(args, family).split(",")):
            B, n, d = (int(v) for v in spec.split("x"))
            r = bench_shape(family, B, n, d, args.windows)
            print(json.dumps(r), flush=True)
            out["shapes"].append(r)
    if args.share_generations > 0:
        for name, objective, bound, tol_fun in (("rastrigin", rastrigin, 5.12, 1e-4), ("rosenbrock", rosenbrock, 5.0, 1e-12),
                                                ("lunacek", lunacek(10), 5.0, 1e-4)):
            r = optimum_share(name, objective, bound, tol_fun, args.share_items, args.share_generations, args.share_every)
            print(json.dumps(r), flush=True)
            out["optimum_share"].append(r)
    print(json.dumps(out["card"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
