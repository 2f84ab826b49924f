"""Functional LM-MA-ES over a batch of B independent searches (default popsize 4 + floor(3 ln D), m the same): milliseconds per
generation (ask + fused evaluation of the built-in Rastrigin + tell) against separable CMA-ES and, up to D = 2048, full-covariance
CMA-ES at the same B and D; peak allocated memory of each; and every LM-MA-ES kernel alone (torch.profiler, CUDA activity, in a
run of its own) with its achieved bytes/s against the bytes it must move, computed from the shapes below.  Warm-up, then windows
that alternate the families; medians and spreads over the windows, with the card's name and power limit read in the same run.

    python scripts/functional_lmmaes_bench.py [--shapes 1024x32,64x1000,8x2048,8x10000,1x100000] [--windows 5] [--out FILE]
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

from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask_and_evaluate, cmaes_tell, lmmaes, lmmaes_ask_and_evaluate,  # noqa: E402
                                                 lmmaes_tell, sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell)
from evotorch_b200.objectives import rastrigin  # noqa: E402
from scripts.functional_cmaes_bench import card, timed  # noqa: E402

DEV = torch.device("cuda")
FAMILIES = {"lmmaes": (lmmaes, lmmaes_ask_and_evaluate, lmmaes_tell), "sepcmaes": (sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell),
            "cmaes": (cmaes, cmaes_ask_and_evaluate, cmaes_tell)}
CMAES_MAX_D = 2048  # beyond, B x D x D covariances and their factorisations make a generation take seconds


def stage_bytes(B: int, n: int, d: int, m: int, k: int) -> dict:
    """Bytes each LM-MA-ES kernel must move per generation, all items, at k vectors in use (float32; z is rebuilt, not read)."""
    tiles, mu = math.ceil(d / 512), n // 2
    f = 4 * B
    return {
        "lmmaes_project_kernel<false>": f * (k * d + tiles * k * n),  # M_k read, the tiles' P written
        "lmmaes_coef_kernel": f * (tiles * k * n + k * k + k * n),  # P partials and G read, beta written
        "lmmaes_write_kernel": f * (k * d + d + n * d),  # M_k and y read, x written
        "lmmaes_project_kernel<true>": f * (mu * d + k * d + d + d + tiles * k * mu),  # mu rows, M_k, y read; S_d and Q partials written
        "lmmaes_recover_kernel": f * (tiles * k * mu + k * k + n + 1 + m),
        "lmmaes_update_kernel": f * (m * d + 3 * d + m * d + 2 * d + tiles * (m * m + 1)),  # M, S_d, y, p read; M', y', p' written
        "lmmaes_finish_kernel": f * (tiles * (m * m + 1) + m * m + 2),
    }


def stages(B: int, d: int, gens: int = 20) -> dict:
    """Each LM-MA-ES kernel's mean time (torch.profiler) over `gens` generations at k = m, and its bytes/s."""
    state = lmmaes(center_init=torch.rand(B, d, device=DEV) * 4 - 2, stdev_init=1.0, objective_sense="min")
    m = state.num_vectors
    state = state._replace(generation=m)  # k = m: every stage at full width
    for _ in range(3):
        v, e = lmmaes_ask_and_evaluate(state, objective=rastrigin)
        state = lmmaes_tell(state, v, e)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(gens):
            v, e = lmmaes_ask_and_evaluate(state, objective=rastrigin)
            state = lmmaes_tell(state, v, e)
        torch.cuda.synchronize()
    times = {}
    for ev in prof.events():
        if "lmmaes_" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
            for key in stage_bytes(1, 2, 2, 1, 1):
                base = key.split("<")[0]
                tmpl = key[len(base):]
                if base in ev.name and (not tmpl or ("<true>" in ev.name) == (tmpl == "<true>")):
                    times.setdefault(key, []).append(ev.device_time_total / 1e3)
    nbytes = stage_bytes(B, state.popsize, d, m, m)
    out = {}
    for key, ts in times.items():
        ms = statistics.mean(ts)
        out[key] = {"ms": ms, "bytes": nbytes[key], "GB_per_s": nbytes[key] / (ms * 1e-3) / 1e9}
    return out


def bench_shape(B: int, d: int, windows: int) -> dict:
    torch.manual_seed(0)
    centers = torch.rand(B, d, device=DEV) * 4 - 2
    res = {"B": B, "D": d}
    runs = {}
    for fam, (make, ask, tell) in FAMILIES.items():
        if fam == "cmaes" and d > CMAES_MAX_D:
            continue
        box = {"s": make(center_init=centers, stdev_init=1.0, objective_sense="min")}

        def step(box=box, ask=ask, tell=tell):
            v, e = ask(box["s"], objective=rastrigin)
            box["s"] = tell(box["s"], v, e)

        runs[fam] = step
        res[f"{fam}_popsize"] = box["s"].popsize
    gens = max(5, min(200, int(2e9 / (B * d * 40))))
    peaks = {}
    for fam, step in runs.items():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        for _ in range(max(3, gens // 5)):
            step()
        torch.cuda.synchronize()
        peaks[fam] = (torch.cuda.max_memory_allocated() - base) / 2**20
    samples = {fam: [] for fam in runs}
    for _ in range(windows):
        for fam, step in runs.items():
            samples[fam].append(timed(step, gens))
    for fam, ms in samples.items():
        res[f"{fam}_ms"] = statistics.median(ms)
        res[f"{fam}_ms_spread"] = [min(ms), max(ms)]
        res[f"{fam}_peak_MiB_above_state"] = peaks[fam]
    res["gens_per_window"] = gens
    res["lmmaes_stages"] = stages(B, d)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1024x32,64x1000,8x2048,8x10000,1x100000")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "shapes": []}
    print(json.dumps(out["card"]), flush=True)
    for shape in a.shapes.split(","):
        B, d = (int(v) for v in shape.split("x"))
        r = bench_shape(B, d, a.windows)
        out["shapes"].append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
