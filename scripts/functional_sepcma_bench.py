"""Functional separable CMA-ES over a batch of B independent searches (N = popsize, D = solution length): milliseconds per
generation of all B searches and peak allocated memory, for
    (a) stored      -- sepcmaes_ask_and_evaluate / sepcmaes_tell on the kernels, the population stored once;
    (b) lazy        -- the same with lazy=True: the population is never stored, the tell rebuilds its rows;
    (c) class loop  -- B CMAES(separable=True) objects stepped one after another on their fused path (timed on a subset of the
                       objects and scaled to B, which the output says);
    (d) torch       -- the module's own batched torch path (sepcmaes_tell's torch branch) on CUDA tensors.
Objectives: the built-in Rastrigin, and a FusedObjective with data (the shifted sphere, one shift per item; in (c) each object
gets its own shift, in (d) it is evaluated by torch ops).  Warm-up, then windows alternating (a)-(d); the median and spread over
the windows are reported, with the card's name and power limit read in the same run.  For (a) the moments pass is also timed
alone with CUDA events, and its achieved bytes/s reported against the bytes it must read: every row with a non-zero weight once,
and the rows with a negative weight a second time for their squared norms.

    python scripts/functional_sepcma_bench.py [--shapes 1024x24x1000,64x200x10000,8x1000x100000,1x100000x4096] [--windows 3] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evotorch_b200 import Problem, ops  # noqa: E402
from evotorch_b200.algorithms import CMAES  # noqa: E402
from evotorch_b200.algorithms.functional import funcsepcmaes as F  # noqa: E402
from evotorch_b200.algorithms.functional import sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell  # noqa: E402
from evotorch_b200.objectives import FusedObjective, rastrigin  # noqa: E402
from scripts.functional_cmaes_bench import card, timed  # noqa: E402

DEV = torch.device("cuda")


def torch_tell(state, x, f):
    """The module's batched torch tell on CUDA tensors (what sepcmaes_tell runs off the kernels)."""
    batch, B, d = F._items(state)
    m, sigma, C, A, s, p_sigma, p_c = F._tell_torch(state, B, state.popsize, d, x.reshape(B, state.popsize, d), f.reshape(B, state.popsize))
    vec = batch + (d,)
    return state._replace(center=m.view(vec), sigma=sigma.view(batch), C=C.view(vec), A=A.view(vec), s=s.view(vec), p_sigma=p_sigma.view(vec),
                          p_c=p_c.view(vec), generation=state.generation + 1)


def moments_rate(state, objective) -> dict:
    """The moments pass of one stored generation alone: ms (CUDA events, median of 20) and bytes/s against the bytes it must read."""
    values, evals = sepcmaes_ask_and_evaluate(state, objective=objective)
    B, n, d = values.shape[0] if values.ndim == 3 else 1, state.popsize, state.center.shape[-1]
    X = values.reshape(B, n, d)
    m, s = state.center.reshape(B, d), state.s.reshape(B, d)
    aw = ops.rank_table_batched(evals.reshape(B, n), False, state.weights)
    rows = int((aw != 0).sum()) + (int((aw < 0).sum()) if state.active else 0)
    ms = []
    for _ in range(22):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.sepcma_moments_batched(X, m, s, aw, state.active)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    t = statistics.median(ms[2:])
    nbytes = rows * d * 4
    return {"ms": t, "rows_read_per_item_row": rows / (B * n), "bytes": nbytes, "GB_per_s": nbytes / (t * 1e-3) / 1e9}


def bench_shape(B: int, n: int, d: int, objective: str, windows: int, class_subset: int) -> dict:
    torch.manual_seed(0)
    centers = torch.rand(B, d, device=DEV) * 4 - 2
    res = {"B": B, "N": n, "D": d, "objective": objective}
    if objective == "rastrigin":
        fused, torch_fn, per_object = rastrigin, rastrigin, [rastrigin] * min(B, class_subset)
    else:
        shifts = torch.rand(B, d, device=DEV) * 2 - 1
        fused = FusedObjective("shifted_sphere", {"s": "(x - o)**2"}, "s", data={"o": shifts})
        single = FusedObjective("shifted_sphere", {"s": "(x - o)**2"}, "s", data={"o": shifts[0].clone()})

        def torch_fn(x):
            return ((x - shifts[:, None, :]) ** 2).sum(-1)

        per_object = [single.with_data(o=shifts[i].clone()) for i in range(min(B, class_subset))]

    def fresh():
        return sepcmaes(center_init=centers, stdev_init=1.0, objective_sense="min", popsize=n)

    box = {"stored": fresh(), "lazy": fresh(), "torch": fresh()}

    def step(lazy):
        key = "lazy" if lazy else "stored"

        def run():
            values, evals = sepcmaes_ask_and_evaluate(box[key], objective=fused, lazy=lazy)
            box[key] = sepcmaes_tell(box[key], values, evals)
        return run

    k = len(per_object)
    searchers = []
    for i in range(k):
        prob = Problem("min", per_object[i], solution_length=d, initial_bounds=(-1, 1), device=DEV, seed=i)
        searchers.append(CMAES(prob, stdev_init=1.0, popsize=n, center_init=centers[i].clone(), separable=True))

    def step_c():
        for s in searchers:
            s.step()

    def step_d():
        st = box["torch"]
        x = st.center[..., None, :] + st.s[..., None, :] * torch.randn(B, n, d, device=DEV)
        box["torch"] = torch_tell(st, x, torch_fn(x))

    runs = {"stored": (step(False), 1.0), "lazy": (step(True), 1.0), "class_loop": (step_c, B / k), "torch_batched": (step_d, 1.0)}
    peak = {}
    for name, (run, _) in runs.items():  # warm-up: module loads, library handles, workspaces
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() - base
    gens = {}
    for name, (run, _) in runs.items():  # about 0.3 s per window
        t = timed(run, 2)
        gens[name] = max(2, min(100, int(300 / max(t, 1e-3))))
    samples = {name: [] for name in runs}
    for _ in range(windows):
        for name, (run, scale) in runs.items():
            if name in box:  # every window starts from the initial state
                box[name] = fresh()
            samples[name].append(timed(run, gens[name]) * scale)
    for name, xs in samples.items():
        res[name] = {"ms_per_generation": statistics.median(xs), "min": min(xs), "max": max(xs), "windows": len(xs), "gens_per_window": gens[name],
                     "extra_peak_allocated_MiB": round(peak[name] / 2**20, 2)}
    res["class_loop"]["timed_objects"] = k
    res["stored_moments"] = moments_rate(fresh(), fused)
    res["finite"] = all(bool(torch.isfinite(s.center).all()) for s in box.values())
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1024x24x1000,64x200x10000,8x1000x100000,1x100000x4096")
    ap.add_argument("--objectives", default="rastrigin,shifted_sphere")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--class-subset", type=int, default=16, help="CMAES objects actually stepped in (c); the time is scaled to B")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("functional_sepcma_bench needs a CUDA device")
    out = {"card": card(), "shapes": []}
    print(json.dumps(out["card"]), flush=True)
    for spec in args.shapes.split(","):
        B, n, d = (int(v) for v in spec.split("x"))
        for objective in args.objectives.split(","):
            if B == 1 and objective != "rastrigin":
                continue  # one item: the data-batched objective is the single search's
            r = bench_shape(B, n, d, objective, args.windows, args.class_subset)
            print(json.dumps(r), flush=True)
            out["shapes"].append(r)
    out["card_after"] = card()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
