"""Functional CMA-ES with restarts over a batch of B independent searches (N = popsize, D = solution length): milliseconds per
generation of all B searches for
    (a) restarts    -- ask (+ fused evaluation), restarts_tell: per-item counters, best ever, criteria and resets on the device;
    (b) plain       -- the same ask, the family's tell and a best-so-far per item kept with torch ops on the host side of the API
                       (the best finite eval of the generation, its row, a torch.where update), which is what users write today;
and the restart stage alone (ops.cma_restart_batched, CUDA events, median of 50 launches, the items not restarting).  Shapes are
those of functional_cmaes_bench.py (cmaes) and functional_sepcma_bench.py (sepcmaes, stored populations).  Finally the share of
items whose best ever reaches f < 1e-8 on 10-D Rastrigin at a fixed generation budget, with and without restarts, at popsize 10 and
100 (tol_fun 1e-4: float32 Rastrigin resolves fitness ranges of ~1e-5 only).  Warm-up,
then windows alternating (a) and (b); medians over the windows, with the card's name and power limit read in the same run.

    python scripts/functional_restart_bench.py [--cmaes 1024x16x32,...] [--sepcmaes 1024x24x1000,...] [--windows 3] [--out FILE]
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
from evotorch_b200.algorithms.functional import (SepCMAESState, cmaes, cmaes_ask_and_evaluate, cmaes_tell, restarts,  # noqa: E402
                                                 restarts_tell, sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell)
from evotorch_b200.objectives import rastrigin  # noqa: E402
from scripts.functional_cmaes_bench import card, timed  # noqa: E402

DEV = torch.device("cuda")


def track_best(best_x, best_f, values, evals):
    """Host-side best-so-far per item with torch ops (minimisation)."""
    f = torch.where(torch.isfinite(evals), evals, math.inf)
    g, i = f.min(-1)
    row = torch.gather(values, -2, i[..., None, None].expand(i.shape + (1, values.shape[-1])))[..., 0, :]
    better = g < best_f
    return torch.where(better[..., None], row, best_x), torch.where(better, g, best_f)


def stage_ms(rs) -> float:
    """The restart stage alone on the state of `rs` after one more generation (no item restarts: thresholds off)."""
    sep = isinstance(rs.search, SepCMAESState)
    ask = sepcmaes_ask_and_evaluate if sep else cmaes_ask_and_evaluate
    values, evals = ask(rs.search, objective=rastrigin)
    B, d = rs.search.center.reshape(-1, rs.search.center.shape[-1]).shape
    n = rs.search.popsize
    s = rs.search
    mat = (B, d) if sep else (B, d, d)
    st = [s.center.reshape(B, d).clone(), s.sigma.reshape(B).clone(), s.p_sigma.reshape(B, d).clone(), s.p_c.reshape(B, d).clone(),
          s.C.reshape(mat).clone(), s.A.reshape(mat).clone(), s.s.reshape(B, d).clone() if sep else None]
    steps = rs.item_generation.reshape(B).clone() + 1
    hist, bx, bf, nr = rs.history.reshape(B, -1).clone(), rs.best_values.reshape(B, d).clone(), rs.best_evals.reshape(B).clone(), rs.num_restarts.reshape(B).clone()
    flags = torch.empty(B, dtype=torch.int32, device=DEV)
    f, X = evals.reshape(B, n).contiguous(), values.reshape(B, n, d).contiguous()
    sig0, lb, ub = rs.stdev_init.reshape(B).contiguous(), rs.lb.reshape(B, d), rs.ub.reshape(B, d)
    ms = []
    for _ in range(55):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.cma_restart_batched(sep, f, X, False, steps, *st, hist, bx, bf, nr, flags, sig0, lb, ub, (None,) * 6, seed=1)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms[5:])


def bench_shape(family: str, B: int, n: int, d: int, windows: int) -> dict:
    torch.manual_seed(0)
    make, ask, tell = (cmaes, cmaes_ask_and_evaluate, cmaes_tell) if family == "cmaes" else (sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell)
    state = make(center_init=torch.rand(B, d, device=DEV) * 4 - 2, stdev_init=1.0, objective_sense="min", popsize=n)
    box = {"rs": restarts(state, lb=-5.12, ub=5.12), "s": state, "bx": torch.full((B, d), math.nan, device=DEV),
           "bf": torch.full((B,), math.inf, device=DEV)}

    def step_a():
        values, evals = ask(box["rs"].search, objective=rastrigin)
        box["rs"] = restarts_tell(box["rs"], values, evals)

    def step_b():
        values, evals = ask(box["s"], objective=rastrigin)
        box["s"] = tell(box["s"], values, evals)
        box["bx"], box["bf"] = track_best(box["bx"], box["bf"], values, evals)

    gens = max(3, min(50, int(2e9 // max(1, B * n * d * (d if family == "cmaes" else 1) * 4))))
    for fn in (step_a, step_b):
        fn()
        fn()
    a_ms, b_ms = [], []
    for _ in range(windows):
        a_ms.append(timed(step_a, gens))
        b_ms.append(timed(step_b, gens))
    return {"family": family, "B": B, "N": n, "D": d, "gens_per_window": gens, "restarts_ms": statistics.median(a_ms),
            "plain_plus_best_ms": statistics.median(b_ms), "restarts_ms_spread": [min(a_ms), max(a_ms)],
            "plain_ms_spread": [min(b_ms), max(b_ms)], "stage_ms": stage_ms(box["rs"])}


def optimum_share(B: int, gens: int, popsize: int) -> dict:
    out = {"objective": "rastrigin", "D": 10, "B": B, "popsize": popsize, "generations": gens, "tol_fun": 1e-4}
    for restart in (True, False):
        torch.manual_seed(123)
        state = cmaes(center_init=torch.rand(B, 10, device=DEV) * 10.24 - 5.12, stdev_init=1.5, objective_sense="min", popsize=popsize)
        if restart:
            rs = restarts(state, lb=-5.12, ub=5.12, tol_fun=1e-4)  # float32 Rastrigin (~10 D) resolves fitness ranges of ~1e-5
            for _ in range(gens):
                rs = restarts_tell(rs, *cmaes_ask_and_evaluate(rs.search, objective=rastrigin))
            best, nr = rs.best_evals, rs.num_restarts.float().mean().item()
        else:
            best, bx = torch.full((B,), math.inf, device=DEV), torch.full((B, 10), math.nan, device=DEV)
            for _ in range(gens):
                values, evals = cmaes_ask_and_evaluate(state, objective=rastrigin)
                state = cmaes_tell(state, values, evals)
                bx, best = track_best(bx, best, values, evals)
            nr = 0.0
        out["with_restarts" if restart else "without_restarts"] = {"share_f_below_1e-8": (best < 1e-8).float().mean().item(),
                                                                  "median_best": best.median().item(), "mean_restarts": nr}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cmaes", default="1024x16x32,256x20x128,64x24x512,8x32x2048")
    ap.add_argument("--sepcmaes", default="1024x24x1000,64x200x10000,8x1000x100000,1x100000x4096")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--share-items", type=int, default=1024)
    ap.add_argument("--share-generations", type=int, default=2000)
    ap.add_argument("--share-popsizes", default="10,100")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("functional_restart_bench.py measures on a CUDA device; none is available")
    out = {"card": card(), "shapes": []}
    for family in ("cmaes", "sepcmaes"):
        for spec in filter(None, getattr(args, family).split(",")):
            B, n, d = (int(v) for v in spec.split("x"))
            r = bench_shape(family, B, n, d, args.windows)
            print(json.dumps(r), flush=True)
            out["shapes"].append(r)
    out["optimum_share"] = []
    for popsize in filter(None, args.share_popsizes.split(",")):
        out["optimum_share"].append(optimum_share(args.share_items, args.share_generations, int(popsize)))
        print(json.dumps(out["optimum_share"][-1]), flush=True)
    print(json.dumps(out["card"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
