"""Functional CMA-ES with the batched evaluation kernel against the torch expression.

    python scripts/functional_cmaes_fused_bench.py [--windows 5] [--gens 10] [--reps 5] [--out results.json]

1. Whole generations at README's `cmaes` shapes (B x popsize x D): `cmaes_ask` + the objective's torch expression + `cmaes_tell`
   against `cmaes_ask_and_evaluate` + `cmaes_tell`, on Rastrigin and on a per-item shifted sphere.  ms per generation and the
   peak memory allocated above the state during one generation.
2. Evaluation alone: a per-item shifted Rosenbrock on (B, N, D) populations, the torch expression against `evaluate_batched`,
   with the read rate 4 B N D bytes over the kernel time.

Times are CUDA-event medians over windows that alternate between the two forms.  The card's name and power limit are read in the
same run and printed with the numbers."""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evotorch_b200 import ops  # noqa: E402
from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_ask_and_evaluate, cmaes_tell  # noqa: E402
from evotorch_b200.objectives import FusedObjective, rastrigin  # noqa: E402

SHAPES = [(1024, 16, 32), (256, 20, 128), (64, 24, 512), (8, 32, 2048)]
EVAL_SHAPES = [(1024, 1000, 1000), (64, 10_000, 1000)]
ROSENBROCK = {"s": "100*((xn - o_n) - (x - o)**2)**2 + (1 - (x - o))**2"}


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [s.strip() for s in out.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power}


def timed(fn, n: int) -> float:
    """ms per call of fn over n calls, by CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def alternate(forms: dict, n: int, windows: int) -> dict:
    """{name: median ms per call} over `windows` windows of n calls per form, the forms alternating."""
    for fn in forms.values():  # warm-up: module loads, compiles, allocator
        fn()
        fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in forms}
    for _ in range(windows):
        for k, fn in forms.items():
            samples[k].append(timed(fn, n))
    return {k: statistics.median(v) for k, v in samples.items()}


def extra_peak_mib(fn) -> float:
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def generations(args) -> list:
    rows = []
    for B, n, D in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(B + D)
        shift = torch.randn(B, D, device="cuda", generator=g)
        objectives = {"rastrigin": rastrigin,
                      "shifted_sphere": FusedObjective("shifted_sphere", sums={"s": "(x - o)**2"}, value="s", data={"o": shift})}
        for oname, obj in objectives.items():
            state0 = cmaes(center_init=torch.randn(B, D, device="cuda", generator=g), stdev_init=1.0, objective_sense="min", popsize=n)
            st = {"torch": state0, "fused": state0}

            def torch_gen():
                values = cmaes_ask(st["torch"])
                st["torch"] = cmaes_tell(st["torch"], values, obj._torch_fn(values))

            def fused_gen():
                values, evals = cmaes_ask_and_evaluate(st["fused"], objective=obj)
                st["fused"] = cmaes_tell(st["fused"], values, evals)

            ms = alternate({"torch": torch_gen, "fused": fused_gen}, args.gens, args.windows)
            mem = {"torch": extra_peak_mib(torch_gen), "fused": extra_peak_mib(fused_gen)}
            row = {"B": B, "popsize": n, "D": D, "objective": oname, "ms_torch": ms["torch"], "ms_fused": ms["fused"],
                   "peak_mib_torch": mem["torch"], "peak_mib_fused": mem["fused"]}
            print(json.dumps(row), flush=True)
            rows.append(row)
    return rows


def evaluation(args) -> list:
    rows = []
    for B, N, D in EVAL_SHAPES:
        g = torch.Generator(device="cuda").manual_seed(N)
        shift = torch.randn(B, D, device="cuda", generator=g)
        obj = FusedObjective("shifted_rosenbrock", sums=ROSENBROCK, value="s", data={"o": shift})
        obj.compile_eval_batched()
        X = torch.randn(B, N, D, device="cuda", generator=g)
        f = torch.empty(B, N, device="cuda")
        ref = obj._torch_fn(X)
        got = ops.evaluate_batched(obj.evok_objective_id, X, seed=1, f=f)
        rel = ((got.double() - ref.double()).abs() / ref.double().abs().clamp_min(1.0)).max().item()
        del ref
        ms = alternate({"torch": lambda: obj._torch_fn(X), "kernel": lambda: ops.evaluate_batched(obj.evok_objective_id, X, seed=1, f=f)},
                       args.reps, args.windows)
        nbytes = 4 * B * N * D
        row = {"B": B, "N": N, "D": D, "ms_torch": ms["torch"], "ms_kernel": ms["kernel"], "read_TBps_kernel": nbytes / ms["kernel"] / 1e9,
               "read_TBps_torch": nbytes / ms["torch"] / 1e9, "max_rel_diff": rel}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del X, f
        torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("this benchmark measures the GPU: no CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    result = {**info, "generations": generations(args), "evaluation": evaluation(args)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
