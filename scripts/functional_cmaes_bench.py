"""Functional CMA-ES over a batch of B independent searches (N = popsize, D = solution length): milliseconds per generation of all
B searches and peak allocated memory, for
    (a) functional  -- cmaes_ask / cmaes_tell on the kernels (one launch per stage for all items);
    (b) class loop  -- B CMAES objects stepped one after another on their fused path (per generation; timed on a subset of the
                       objects and scaled to B, which the output says);
    (c) torch       -- the same algorithm as batched torch ops (bmm, argsort, cholesky) written here.
The objective is the sphere (evaluated by torch ops in (a) and (c), by the fused sampler kernel in (b)).  Warm-up, then windows
alternating (a), (b), (c); the median and the spread over the windows are reported, with the card's name and power limit.

    python scripts/functional_cmaes_bench.py [--shapes 1024x16x32,256x20x128,64x24x512,8x32x2048] [--windows 5] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evotorch_b200 import Problem  # noqa: E402
from evotorch_b200.algorithms import CMAES  # noqa: E402
from evotorch_b200.algorithms.cmaes import cmaes_hyperparameters  # noqa: E402
from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_tell  # noqa: E402
from evotorch_b200.objectives import sphere  # noqa: E402

DEV = torch.device("cuda")


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = (v.strip() for v in q.split(","))
    except Exception as e:  # the number is still reported, without the power limit
        out["power_limit"] = f"unread ({type(e).__name__})"
    return out


# ------------------------------------------------------------------------------------------------ (c) batched torch ops
class TorchCMAES:
    """Full-covariance CMA-ES for B items with batched torch ops; the arithmetic of CMAES's op-by-op generation."""

    def __init__(self, centers: torch.Tensor, sigma: float, n: int):
        B, d = centers.shape
        self.hp = cmaes_hyperparameters(d, n, dtype=centers.dtype, device=centers.device)
        self.m, self.sigma = centers.clone(), torch.full((B,), sigma, device=centers.device)
        self.C = torch.eye(d, device=centers.device).expand(B, d, d).contiguous()
        self.A = self.C.clone()
        self.p_sigma, self.p_c = torch.zeros_like(self.m), torch.zeros_like(self.m)
        self.gen = 0

    def step(self, fn) -> None:
        hp, (B, d), n = self.hp, self.m.shape, self.hp.popsize
        z = torch.randn(B, n, d, device=self.m.device)
        y = torch.bmm(z, self.A.mT)
        x = self.m[:, None, :] + self.sigma[:, None, None] * y
        f = fn(x)
        ranks = torch.empty(B, n, dtype=torch.int64, device=f.device).scatter_(
            -1, torch.argsort(f, dim=-1, stable=True), torch.arange(n, device=f.device).expand(B, n).contiguous())
        aw = hp.weights[ranks]
        wp = aw.clamp_min(0)
        local, shaped = torch.bmm(wp[:, None, :], z)[:, 0], torch.bmm(wp[:, None, :], y)[:, 0]
        self.m = self.m + hp.c_m * self.sigma[:, None] * shaped
        self.p_sigma = (1 - hp.c_sigma) * self.p_sigma + hp.variance_discount_sigma * local
        pn = torch.linalg.vector_norm(self.p_sigma, dim=-1)
        self.sigma = self.sigma * torch.exp((hp.c_sigma / hp.damp_sigma) * (pn / hp.unbiased_expectation - 1))
        h = ((pn**2 / (1 - (1 - hp.c_sigma) ** (2 * self.gen + 1)) / d) - 1 < 1 + 4.0 / (d + 1)).float()
        self.p_c = (1 - hp.c_c) * self.p_c + (h * hp.variance_discount_c)[:, None] * shaped
        w = torch.where(aw > 0, aw, d * aw / (z * z).sum(-1))
        c1a = hp.c_1 * (1 - (1 - h**2) * hp.c_c * (2 - hp.c_c))
        pc = ((hp.c_1 / (c1a + 1e-23)) ** 0.5)[:, None] * self.p_c
        self.C = (self.C + c1a[:, None, None] * (pc[:, :, None] * pc[:, None, :] - self.C)
                  + hp.c_mu * (torch.bmm(y.mT * w[:, None, :], y) - hp.weights_sum * self.C))
        if (self.gen + 1) % hp.decompose_C_freq == 0:
            self.A, _ = torch.linalg.cholesky_ex(self.C, check_errors=False)
        self.gen += 1


def sphere_torch(x):
    return (x * x).sum(-1)


def timed(run, gens: int) -> float:
    """ms per generation of `run` over `gens` generations (host clock around work that ends in a device synchronise)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(gens):
        run()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / gens


def bench_shape(B: int, n: int, d: int, windows: int, class_subset: int) -> dict:
    torch.manual_seed(0)
    centers = torch.randn(B, d, device=DEV)
    res = {"B": B, "N": n, "D": d}

    # (a) functional on the kernels
    box = {"s": cmaes(center_init=centers, stdev_init=1.0, objective_sense="min", popsize=n)}

    def step_a():
        x = cmaes_ask(box["s"])
        box["s"] = cmaes_tell(box["s"], x, sphere_torch(x))

    # (b) CMAES objects on their fused path: a subset, scaled to B
    k = min(B, class_subset)
    searchers = []
    for i in range(k):
        prob = Problem("min", sphere, solution_length=d, initial_bounds=(-1, 1), device=DEV, seed=i)
        searchers.append(CMAES(prob, stdev_init=1.0, popsize=n, center_init=centers[i].clone()))

    def step_b():
        for s in searchers:
            s.step()

    # (c) batched torch ops
    tc = TorchCMAES(centers, 1.0, n)

    def step_c():
        tc.step(sphere_torch)

    runs = {"functional": (step_a, 1.0), "class_loop": (step_b, B / k), "torch_batched": (step_c, 1.0)}
    peak = {}
    for name, (run, _) in runs.items():  # warm-up: module loads, library handles, workspaces
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() - base
    gens = {}
    for name, (run, _) in runs.items():  # about 0.3 s per window
        t = timed(run, 2)
        gens[name] = max(2, min(200, int(300 / max(t, 1e-3))))
    # every window of (a) and (c) starts from the initial state, so that no window runs on a search that has converged to zero
    resets = {"functional": lambda: box.update(s=cmaes(center_init=centers, stdev_init=1.0, objective_sense="min", popsize=n)),
              "torch_batched": lambda: tc.__init__(centers, 1.0, n)}
    samples = {name: [] for name in runs}
    for _ in range(windows):
        for name, (run, scale) in runs.items():
            if name in resets:
                resets[name]()
            samples[name].append(timed(run, gens[name]) * scale)
    for name, xs in samples.items():
        res[name] = {"ms_per_generation": statistics.median(xs), "min": min(xs), "max": max(xs), "windows": len(xs), "gens_per_window": gens[name],
                     "extra_peak_allocated_MiB": round(peak[name] / 2**20, 2)}
    res["class_loop"]["timed_objects"] = k
    finite = bool(torch.isfinite(box["s"].center).all()) and bool(torch.isfinite(tc.m).all())
    res["finite"] = finite
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1024x16x32,256x20x128,64x24x512,8x32x2048")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--class-subset", type=int, default=32, help="CMAES objects actually stepped in (b); the time is scaled to B")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("functional_cmaes_bench needs a CUDA device")
    out = {"card": card(), "shapes": []}
    for spec in args.shapes.split(","):
        B, n, d = (int(v) for v in spec.split("x"))
        r = bench_shape(B, n, d, args.windows, args.class_subset)
        print(json.dumps(r), flush=True)
        out["shapes"].append(r)
    print(json.dumps(out["card"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
