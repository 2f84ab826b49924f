"""IPOP restarts of the functional CMA-ES families (padded populations) over a batch of B searches (N = lambda_0, D = solution
length), measured against plain restarts:
    (a) ms per generation of all B items (ask + fused evaluation + restarts_tell) for IPOP with the ladder N, 2N, ..., 8N and the
        items spread over every tier, against plain restarts at popsize N and at popsize 8N.  Windows alternate the three; medians.
    (b) the tiered stages alone (rank table, restart stage) against the untiered ones at the padded size, CUDA events, median of
        50 launches.
    (c) the share of items whose best ever reaches f < 1e-8 on 10-D Rastrigin (tol_fun 1e-4) against the mean evaluations per
        item, for IPOP from popsize 10 (x2, max 640) and for plain restarts at popsize 10 and 100, at equal evaluation budgets.
The ask draws and evaluates all 8N rows of every IPOP item (the pad rows included), which (a) measures.  The card's name and power
limit are read in the same run.

    python scripts/functional_ipop_bench.py [--cmaes 1024x16x32,...] [--sepcmaes 1024x24x1000,...] [--windows 3] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
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

DEV = torch.device("cuda")
MULT = 8  # the top of the ladder, in multiples of lambda_0


def _events(fn, reps: int = 55) -> float:
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms[5:])


def bench_shape(family: str, B: int, n: int, d: int, windows: int) -> dict:
    torch.manual_seed(0)
    make, ask = (cmaes, cmaes_ask_and_evaluate) if family == "cmaes" else (sepcmaes, sepcmaes_ask_and_evaluate)
    centre = torch.rand(B, d, device=DEV) * 4 - 2
    big = n * MULT
    ipop = restarts(make(center_init=centre, stdev_init=1.0, objective_sense="min", popsize=n), lb=-5.12, ub=5.12, popsize_multiplier=2,
                    max_popsize=big)
    K = len(ipop.ladder.popsizes)
    ipop = ipop._replace(tier=(torch.arange(B, device=DEV) % K).to(torch.int32))  # every tier present
    box = {"ipop": ipop, "small": restarts(make(center_init=centre, stdev_init=1.0, objective_sense="min", popsize=n), lb=-5.12, ub=5.12),
           "big": restarts(make(center_init=centre, stdev_init=1.0, objective_sense="min", popsize=big), lb=-5.12, ub=5.12)}

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
    out = {"family": family, "B": B, "N": n, "max_popsize": big, "ladder": list(ipop.ladder.popsizes), "D": d, "gens_per_window": gens}
    for k, label in (("ipop", "ipop_ms"), ("small", f"plain_popsize_{n}_ms"), ("big", f"plain_popsize_{big}_ms")):
        out[label] = statistics.median(ms[k])
        out[label + "_spread"] = [min(ms[k]), max(ms[k])]
    out.update(stages_ms(box["ipop"], ask))
    return out


def stages_ms(rs, ask) -> dict:
    """The tiered rank table and restart stage against the untiered ones on the same padded (B, max_popsize) fitnesses."""
    s = rs.search
    sep = isinstance(s, SepCMAESState)
    values, evals = ask(s, objective=rastrigin)
    B, d = s.center.reshape(-1, s.center.shape[-1]).shape
    n = s.popsize
    f, X = evals.reshape(B, n).contiguous(), values.reshape(B, n, d).contiguous()
    lad, tier = rs.ladder, rs.tier.reshape(B).contiguous()
    out = {"rank_tiered_ms": _events(lambda: ops.rank_table_batched(f, False, lad.weights, tier=tier, counts=lad.counts)),
           "rank_untiered_ms": _events(lambda: ops.rank_table_batched(f, False, lad.weights[-1].contiguous()))}
    mat = (B, d) if sep else (B, d, d)
    st = [s.center.reshape(B, d).clone(), s.sigma.reshape(B).clone(), s.p_sigma.reshape(B, d).clone(), s.p_c.reshape(B, d).clone(),
          s.C.reshape(mat).clone(), s.A.reshape(mat).clone(), s.s.reshape(B, d).clone() if sep else None]
    steps = rs.item_generation.reshape(B).clone() + 1
    r = [rs.history.reshape(B, -1).clone(), rs.best_values.reshape(B, d).clone(), rs.best_evals.reshape(B).clone(), rs.num_restarts.reshape(B).clone()]
    flags = torch.empty(B, dtype=torch.int32, device=DEV)
    sig0, lb, ub = rs.stdev_init.reshape(B).contiguous(), rs.lb.reshape(B, d), rs.ub.reshape(B, d)
    t2, ne = tier.clone(), rs.num_evaluations.reshape(B).clone()
    args = (sep, f, X, False, steps, *st, *r, flags, sig0, lb, ub, (None,) * 6)
    out["restart_tiered_ms"] = _events(lambda: ops.cma_restart_batched(*args, seed=1, tier=t2, tier_counts=lad.counts, tier_history=lad.history,
                                                                       num_evaluations=ne))
    out["restart_untiered_ms"] = _events(lambda: ops.cma_restart_batched(*args, seed=1))
    return out


def optimum_share(B: int, gens: int, every: int) -> dict:
    """Share at the optimum against mean evaluations per item: IPOP checkpoints every `every` generations, then plain restarts at
    popsize 10 and 100 read at the same evaluation budgets."""
    def start(popsize, **kw):
        torch.manual_seed(123)
        state = cmaes(center_init=torch.rand(B, 10, device=DEV) * 10.24 - 5.12, stdev_init=1.5, objective_sense="min", popsize=popsize)
        return restarts(state, lb=-5.12, ub=5.12, tol_fun=1e-4, **kw)

    rs, curve = start(10, popsize_multiplier=2, max_popsize=640), []
    for g in range(1, gens + 1):
        rs = restarts_tell(rs, *cmaes_ask_and_evaluate(rs.search, objective=rastrigin))
        if g % every == 0:
            curve.append({"generations": g, "mean_evaluations": rs.num_evaluations.double().mean().item(),
                          "share": (rs.best_evals < 1e-8).float().mean().item(), "mean_tier": rs.tier.float().mean().item()})
    out = {"objective": "rastrigin", "D": 10, "B": B, "tol_fun": 1e-4, "ipop": curve}
    for popsize in (10, 100):
        rs, pts, g = start(popsize), [], 0
        for point in curve:
            while (g + 1) * popsize <= point["mean_evaluations"]:
                rs = restarts_tell(rs, *cmaes_ask_and_evaluate(rs.search, objective=rastrigin))
                g += 1
            pts.append({"evaluations": g * popsize, "share": (rs.best_evals < 1e-8).float().mean().item()})
        out[f"plain_popsize_{popsize}"] = pts
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
        raise SystemExit("functional_ipop_bench.py measures on a CUDA device; none is available")
    out = {"card": card(), "shapes": []}
    for family in ("cmaes", "sepcmaes"):
        for spec in filter(None, getattr(args, family).split(",")):
            B, n, d = (int(v) for v in spec.split("x"))
            r = bench_shape(family, B, n, d, args.windows)
            print(json.dumps(r), flush=True)
            out["shapes"].append(r)
    if args.share_generations > 0:
        out["optimum_share"] = optimum_share(args.share_items, args.share_generations, args.share_every)
        print(json.dumps(out["optimum_share"]), flush=True)
    print(json.dumps(out["card"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
