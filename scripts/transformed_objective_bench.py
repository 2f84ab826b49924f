"""Objectives of the transformed row y = M (x - o): what the transform costs and what it buys.

    python scripts/transformed_objective_bench.py [--windows 5] [--gens 20] [--search-items 512] [--out FILE]

(1) Evaluation alone (CUDA events), rotated Rastrigin with a per-item rotation M_b and offset o_b, at B x n x D in
    1024x16x10, 1024x16x40, 256x20x96 (fused path: D <= 96) and 256x20x128, 64x24x512, 8x32x2048, 64x1000x1000 (GEMM path), comparing on
    the same rows (a) the transformed kernels, (b) torch (`torch.matmul` then the torch function, default matmul settings) and
    (c) the untransformed fused evaluation of the same expression on x (the objective without the transform: what the transform
    adds).  Windows alternate (a), (b), (c); medians over the windows.  The transform's achieved rate counts 2 n D^2 FLOP per item
    over the time of (a), against the FP32 peak (67 TFLOP/s) on the fused path and the TF32 peak (495 TFLOP/s) on the GEMM path
    of the H100 SXM data sheet.
(2) Generations: ms per generation of cmaes_ask_and_evaluate + cmaes_tell on rotated against unrotated Rastrigin (the identity
    transform has the same cost as any other, so the unrotated one is the objective without a transform) at the four CMA-ES
    shapes of README, B x N x D = 1024x16x32, 256x20x128, 64x24x512, 8x32x2048.
(3) Search outcome: the success shares of the search-level check (rotated ellipsoid of condition 1e6, D = 10, f < 1e-4 within
    600 generations) for the full and separable families, rotated and unrotated, at --search-items items.
The card's name and power limit are read in the same run.  One JSON object is printed (and written to --out).
"""

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask_and_evaluate, cmaes_tell, sepcmaes,  # noqa: E402
                                                 sepcmaes_ask_and_evaluate, sepcmaes_tell)
from evotorch_b200.objectives import FusedObjective  # noqa: E402

DEV = torch.device("cuda")
CUTOFF = 96  # the largest D of the fused path (EVOK_TRANSFORM_FUSED_MAX_D)
EVAL_SHAPES = [(1024, 16, 10), (1024, 16, 40), (256, 20, 96), (256, 20, 128), (64, 24, 512), (8, 32, 2048), (64, 1000, 1000)]
GEN_SHAPES = [(1024, 16, 32), (256, 20, 128), (64, 24, 512), (8, 32, 2048)]
RASTRIGIN_Y = dict(sums={"s": "y**2 - 10 * cos(2 * pi * y)"}, value="10 * D + s")
RASTRIGIN_X = dict(sums={"s": "x**2 - 10 * cos(2 * pi * x)"}, value="10 * D + s")
ELLIPSOID_Y = dict(sums={"s": "10**(6 * j / maximum(D - 1, 1)) * y**2"}, value="s")


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = (v.strip() for v in q.split(","))
    except Exception as e:  # the number is still reported, without the power limit
        out["power_limit"] = f"unread ({type(e).__name__})"
    return out


def rotations(B: int, D: int, seed: int = 0) -> tuple:
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = torch.linalg.qr(torch.randn(B, D, D, device=DEV, generator=g))[0].contiguous()
    o = 8 * torch.rand(B, D, device=DEV, generator=g) - 4
    return M, o


def window_ms(fn, calls: int) -> float:
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / calls


def timed(fns: dict, windows: int, min_window_ms: float = 200.0) -> dict:
    """Median ms per call of each fn over `windows` windows that alternate the fns, each window long enough to time."""
    calls = {}
    for k, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        t = window_ms(fn, 3)
        calls[k] = max(3, int(min_window_ms / max(t, 1e-3)))
    res = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            res[k].append(window_ms(fn, calls[k]))
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in res.items()}


def bench_eval(B: int, n: int, D: int, windows: int) -> dict:
    M, o = rotations(B, D)
    obj = FusedObjective("rot_rastrigin", transform=(M, o), **RASTRIGIN_Y)
    plain = FusedObjective("rastrigin_x", **RASTRIGIN_X)
    X = (o[:, None, :] + torch.randn(B, n, D, device=DEV)).contiguous()
    a, b, c = obj.evaluate_batched(X, seed=1), obj._torch_fn(X), plain.evaluate_batched(X, seed=1)
    r = timed({"transformed": lambda: obj.evaluate_batched(X, seed=1), "torch": lambda: obj._torch_fn(X),
               "untransformed_fused": lambda: plain.evaluate_batched(X, seed=1)}, windows)
    flop = 2.0 * B * n * D * D
    t = r["transformed"]["median_ms"] * 1e-3
    fused = D <= CUTOFF
    peak = 67e12 if fused else 495e12
    return {"shape": f"{B}x{n}x{D}", "path": "fused" if fused else "gemm", **{k: v["median_ms"] for k, v in r.items()}, "spread": r,
            "transform_tflops": flop / t / 1e12, "share_of_peak": flop / t / peak, "peak": "FP32 67 TFLOP/s" if fused else "TF32 495 TFLOP/s",
            "max_rel_diff_vs_torch": ((a - b).abs() / b.abs().clamp_min(1)).max().item(), "untransformed_vs_transformed_values_differ": bool((a != c).any())}


def bench_generations(B: int, n: int, D: int, gens: int, windows: int) -> dict:
    M, o = rotations(B, D, 1)
    rot = FusedObjective("rot_rastrigin", transform=(M, o), **RASTRIGIN_Y)
    unrot = rot.with_data(transform=(torch.eye(D, device=DEV).expand(B, D, D).contiguous(), o))
    out = {}
    for name, obj in (("rotated", rot), ("unrotated", unrot)):
        box = {"s": cmaes(center_init=o.clone(), stdev_init=1.0, objective_sense="min", popsize=n)}

        def gen(box=box, obj=obj):
            values, evals = cmaes_ask_and_evaluate(box["s"], objective=obj)
            box["s"] = cmaes_tell(box["s"], values, evals)

        out[name] = gen
    r = timed({k: (lambda g=g: [g() for _ in range(gens)]) for k, g in out.items()}, windows)
    return {"shape": f"{B}x{n}x{D}", **{k: v["median_ms"] / gens for k, v in r.items()}}


def search_shares(B: int) -> dict:
    D, G, tau = 10, 600, 1e-4
    torch.manual_seed(0)
    R = torch.linalg.qr(torch.randn(B, D, D, dtype=torch.float64))[0].float().to(DEV)
    o = (8 * torch.rand(B, D) - 4).to(DEV)
    rot = FusedObjective("rot_ell", transform=(R, o), **ELLIPSOID_Y)
    unrot = rot.with_data(transform=(torch.eye(D, device=DEV).expand(B, D, D).contiguous(), o))
    out = {}
    for fam, (make, ask, tell) in (("full", (cmaes, cmaes_ask_and_evaluate, cmaes_tell)), ("separable", (sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell))):
        for k, obj in (("rotated", rot), ("unrotated", unrot)):
            s = make(center_init=torch.zeros(B, D, device=DEV), stdev_init=3.0, objective_sense="min")
            best = torch.full((B,), math.inf, device=DEV)
            for _ in range(G):
                values, evals = ask(s, objective=obj)
                s = tell(s, values, evals)
                best = torch.fmin(best, evals.min(-1).values)
            out[f"{fam}_{k}"] = (best < tau).float().mean().item()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--gens", type=int, default=20)
    ap.add_argument("--search-items", type=int, default=512)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "evaluation": [], "generations": []}
    for B, n, D in EVAL_SHAPES:
        res["evaluation"].append(bench_eval(B, n, D, a.windows))
        print(json.dumps(res["evaluation"][-1]), flush=True)
    for B, n, D in GEN_SHAPES:
        res["generations"].append(bench_generations(B, n, D, a.gens, a.windows))
        print(json.dumps(res["generations"][-1]), flush=True)
    res["search_shares"] = search_shares(a.search_items)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
