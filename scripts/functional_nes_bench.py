"""Functional XNES and SNES over a batch of B independent searches (default popsize 4 + floor(3 ln D)): milliseconds per generation
(ask + fused evaluation of the built-in Rastrigin + tell), medians and spreads over windows that alternate the candidates, with
the card's name and power limit read in the same run.

XNES at each B x D: the kernels; the batched torch path on CUDA (a float64 state: `torch.matrix_exp` and friends); B `XNES`
objects on the same card (a subset of them timed, scaled to B); functional `cmaes` at the same shapes.  Also the XNES tell kernel
alone (CUDA events around repeated launches) with its FLOP count from the shapes, and the relative error of the exponential pair
against float64 (scipy) at the sizes of the tests.  SNES at each B x D: the kernels against B `SNES` objects.

    python scripts/functional_nes_bench.py [--xnes 1024x8,1024x32,256x64,64x96] [--snes 1024x1000,64x10000] [--windows 5] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evotorch_b200 import Problem, ops  # noqa: E402
from evotorch_b200.algorithms import SNES, XNES  # noqa: E402
from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask_and_evaluate, cmaes_tell, snes, snes_ask_and_evaluate, snes_tell,  # noqa: E402
                                                 xnes, xnes_ask_and_evaluate, xnes_tell)
from evotorch_b200.objectives import rastrigin  # noqa: E402
from scripts.functional_cmaes_bench import card, timed  # noqa: E402

DEV = torch.device("cuda")


def functional(make, ask, tell, B, d, dtype=torch.float32, **kw):
    box = {"s": make(center_init=(torch.rand(B, d, device=DEV) * 4 - 2).to(dtype), stdev_init=1.0, objective_sense="min", **kw)}

    def step():
        v, e = ask(box["s"], objective=rastrigin)
        box["s"] = tell(box["s"], v, e)

    return step


def objects(cls, B, d, subset):
    """step() of `subset` searcher objects on their own problems, and the factor that scales its time to B objects."""
    k = min(B, subset)
    algs = []
    for i in range(k):
        prob = Problem("min", rastrigin, initial_bounds=(-2, 2), solution_length=d, device=DEV, seed=i)
        algs.append(cls(prob, stdev_init=1.0))

    def step():
        for a in algs:
            a.step()

    return step, B / k


def launches(step) -> int:
    """libevok launches of one generation, after a warm one."""
    step()
    before = ops.launch_count()
    step()
    torch.cuda.synchronize()
    return ops.launch_count() - before


def windows(cands: dict, gens: int, n_windows: int) -> dict:
    """{name: (median ms per generation, spread)} over windows that alternate the candidates; cands: name -> (step, scale)."""
    for step, _ in cands.values():  # warm-up: every shape, module and workspace
        for _ in range(3):
            step()
    times = {name: [] for name in cands}
    for _ in range(n_windows):
        for name, (step, scale) in cands.items():
            times[name].append(timed(step, gens) * scale)
    return {name: {"ms_per_gen": statistics.median(t), "min": min(t), "max": max(t)} for name, t in times.items()}


def tell_kernel(B, d, reps=50) -> dict:
    """The XNES tell kernel alone (CUDA events over `reps` launches) and its FLOP count: z (2 n D^2), G (2 n D^2 + n D), the
    exponential pair (2 D^3 per product: 10 + 2 s products), mu' (2 D^2), A' and A_inv' (4 D^3)."""
    s = xnes(center_init=torch.rand(B, d, device=DEV) * 4 - 2, stdev_init=1.0, objective_sense="min")
    n = s.popsize
    x = s.center[:, None, :] + torch.randn(B, n, d, device=DEV)
    w = ops.rank_batched(rastrigin(x), "nes", False)
    ops.weights_adjust_batched_(w, 1)
    for _ in range(3):
        ops.xnes_tell_batched(x, w, s.center, s.A, s.A_inv, 1.0, s.stdev_learning_rate)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        ops.xnes_tell_batched(x, w, s.center, s.A, s.A_inv, 1.0, s.stdev_learning_rate)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    flops = B * (4 * n * d * d + n * d + 10 * 2 * d**3 + 2 * d * d + 4 * d**3)  # s = 0 at the default eta_A
    return {"B": B, "D": d, "N": n, "ms": ms, "flop_per_call": flops, "gflop_per_s": flops / ms / 1e6}


def expm_errors() -> dict:
    """Largest Frobenius error of the exponential pair relative to |expm(+-S) - I| (scipy, float64), per D and |S|_2 (as in the
    tests)."""
    import scipy.linalg

    out = {}
    for d in (1, 2, 17, 64, 96):
        for norm2 in (1e-7, 1e-3, 0.5, 4.0, 40.0):
            g = torch.Generator().manual_seed(0)
            Q = torch.linalg.qr(torch.randn(4, d, d, generator=g, dtype=torch.float64))[0]
            lam = 2 * torch.rand(4, d, generator=g, dtype=torch.float64) - 1
            S = (Q * (lam / lam.abs().amax(-1, keepdim=True) * norm2)[:, None, :]) @ Q.mT
            S = (0.5 * (S + S.mT)).float()
            Fp, Fm = (F.double().cpu().numpy() for F in ops.sym_expm_pair_batched(S.to(DEV)))
            err = 0.0
            for b in range(4):
                s = S[b].double().numpy()
                for F, E in ((Fp[b], scipy.linalg.expm(s)), (Fm[b], scipy.linalg.expm(-s))):
                    ref = E - np.eye(d)
                    err = max(err, np.linalg.norm(F - ref) / np.linalg.norm(ref))
            out[f"D={d},|S|={norm2:g}"] = err
    return out


def shapes(text: str) -> list:
    return [tuple(int(v) for v in s.split("x")) for s in text.split(",") if s]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--xnes", default="1024x8,1024x32,256x64,64x96")
    ap.add_argument("--snes", default="1024x1000,64x10000")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--subset", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": card(), "xnes": [], "xnes_tell_kernel": [], "snes": []}
    for B, d in shapes(a.xnes):
        obj_step, scale = objects(XNES, B, d, a.subset)
        cands = {"kernels": (functional(xnes, xnes_ask_and_evaluate, xnes_tell, B, d), 1.0),
                 "torch_float64": (functional(xnes, xnes_ask_and_evaluate, xnes_tell, B, d, dtype=torch.float64), 1.0),
                 "objects": (obj_step, scale),
                 "cmaes_kernels": (functional(cmaes, cmaes_ask_and_evaluate, cmaes_tell, B, d), 1.0)}
        row = {"B": B, "D": d, "N": 4 + int(math.floor(3 * math.log(d))), "launches_per_gen": launches(cands["kernels"][0]),
               **windows(cands, a.gens, a.windows)}
        res["xnes"].append(row)
        print(json.dumps(row), flush=True)
        res["xnes_tell_kernel"].append(tell_kernel(B, d))
        print(json.dumps(res["xnes_tell_kernel"][-1]), flush=True)
    for B, d in shapes(a.snes):
        obj_step, scale = objects(SNES, B, d, a.subset)
        cands = {"kernels": (functional(snes, snes_ask_and_evaluate, snes_tell, B, d), 1.0),
                 "kernels_lazy": (functional(snes, lambda s, objective: snes_ask_and_evaluate(s, objective=objective, lazy=True), snes_tell, B, d), 1.0),
                 "objects": (obj_step, scale)}
        row = {"B": B, "D": d, "N": 4 + int(math.floor(3 * math.log(d))), "launches_per_gen": launches(cands["kernels"][0]),
               "launches_per_gen_lazy": launches(cands["kernels_lazy"][0]), **windows(cands, a.gens, a.windows)}
        res["snes"].append(row)
        print(json.dumps(row), flush=True)
    res["expm_relative_errors"] = expm_errors()
    print(json.dumps(res["expm_relative_errors"]), flush=True)
    print(json.dumps(res["card"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
