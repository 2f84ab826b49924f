"""What noise (rand() / randn()) in a FusedObjective costs, and what it buys over a torch callable:
    python scripts/noisy_objective_bench.py [--gens K] [--warmup W] [--rounds R] [--pgpe N D] [--torch-pgpe N D] [--lazy-pgpe N D]
                                            [--lazy-gens K] [--functional B N D] [--only NAME ...]
PGPE (symmetric, ClipUp) at --pgpe (default 1 000 000 x 10 000), each noisy objective against its noise-free fused twin:
  - F7                    sum (j + 1) x^4 + rand()                       (one draw per row)
  - BBOB-style Rastrigin  (10 D + sum x^2 - 10 cos 2 pi x) exp(0.01 randn())  (one draw per row)
  - input-noise sphere    sum (x + 0.1 randn())^2                        (one draw per row and column)
The same three fused against torch callables drawing with torch.rand / torch.randn at --torch-pgpe (default 200 000 x 10 000).
The input-noise sphere against its twin on the lazy population at --lazy-pgpe (default 1 000 000 x 100 000), with the peak
allocated memory of every window.  Functional PGPE with the input-noise sphere at --functional (default 1024 x 1000 x 1000): the
fused sampler with a stored and with a lazy population against `pgpe_ask` followed by the torch expression, with the peak memory.
The windows of a pair alternate, R rounds, each after W warm-up generations, timed with CUDA events and ended by a synchronise;
sampler_ms is the fused kernel's CUDA-event time in the last round (scripts/fused_objective_bench.py has the window functions).
Needs a GPU; prints the card and its power limit with one JSON line."""

import argparse
import gc
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fused_objective_bench import card, pair, pgpe, window  # noqa: E402

from evotorch_b200 import Problem  # noqa: E402
from evotorch_b200.algorithms import PGPE  # noqa: E402
from evotorch_b200.algorithms.functional import pgpe as func_pgpe  # noqa: E402
from evotorch_b200.algorithms.functional import pgpe_ask, pgpe_ask_and_evaluate, pgpe_tell  # noqa: E402
from evotorch_b200.objectives import FusedObjective  # noqa: E402

SPECS = {
    "f7": (dict(sums={"s": "(j + 1) * x**4"}, value="s + rand()"), dict(sums={"s": "(j + 1) * x**4"}, value="s")),
    "bbob_rastrigin": (dict(sums={"s": "x**2 - 10 * cos(2 * pi * x)"}, value="(10 * D + s) * exp(0.01 * randn())"),
                       dict(sums={"s": "x**2 - 10 * cos(2 * pi * x)"}, value="10 * D + s")),
    "input_noise_sphere": (dict(sums={"s": "(x + 0.1 * randn())**2"}, value="s"), dict(sums={"s": "x**2"}, value="s")),
}


def _vectorized(fn):
    fn.__evotorch_vectorized__ = True
    return fn


TORCH = {
    "f7": _vectorized(lambda x: ((torch.arange(1, x.shape[-1] + 1, device=x.device, dtype=x.dtype) * x**4).sum(-1)
                                 + torch.rand(x.shape[:-1], device=x.device, dtype=x.dtype))),
    "bbob_rastrigin": _vectorized(lambda x: ((10 * x.shape[-1] + (x**2 - 10 * torch.cos(2 * math.pi * x)).sum(-1))
                                             * torch.exp(0.01 * torch.randn(x.shape[:-1], device=x.device, dtype=x.dtype)))),
    "input_noise_sphere": _vectorized(lambda x: ((x + 0.1 * torch.randn_like(x)) ** 2).sum(-1)),
}


def pgpe_lazy(objective, n: int, d: int):
    prob = Problem("min", objective, initial_bounds=(-5, 5), solution_length=d, device="cuda", seed=1, lazy_population=True)
    return PGPE(prob, popsize=n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)


def lazy_pair(a, b, n: int, d: int, args) -> dict:
    """`pair` on the lazy population, with the peak allocated memory of every window."""
    out = {label: {"gens_per_s": [], "peak_allocated_gib": []} for label, _ in (a, b)}
    for _ in range(args.rounds):
        for label, objective in (a, b):
            s = pgpe_lazy(objective, n, d)
            for _ in range(args.warmup):
                s.step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            out[label]["gens_per_s"].append(round(window(s, args.lazy_gens), 3))
            out[label]["peak_allocated_gib"].append(round(torch.cuda.max_memory_allocated() / 2**30, 3))
            del s
            gc.collect()
            torch.cuda.empty_cache()
    return {"size": [n, d], **out}


def functional(B: int, n: int, d: int, fused, torch_fn, args) -> dict:
    """Generations per second and peak allocated GiB of functional PGPE on B searches of one objective."""
    fused.compile_batched()

    def generation(st, variant):
        if variant == "torch":
            values = pgpe_ask(st, popsize=n)
            evals = torch_fn(values)
        else:
            values, evals = pgpe_ask_and_evaluate(st, popsize=n, objective=fused, lazy=variant == "fused_lazy")
        return pgpe_tell(st, values, evals)

    out = {v: {"gens_per_s": [], "peak_allocated_gib": []} for v in ("fused_stored", "fused_lazy", "torch")}
    for _ in range(args.rounds):
        for variant in out:
            st = func_pgpe(center_init=torch.full((B, d), 3.0, device="cuda"), center_learning_rate=0.3, stdev_learning_rate=0.1,
                           objective_sense="min", stdev_init=1.0)
            for _ in range(args.warmup):
                st = generation(st, variant)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.gens):
                st = generation(st, variant)
            b.record()
            torch.cuda.synchronize()
            out[variant]["gens_per_s"].append(round(args.gens / (a.elapsed_time(b) / 1e3), 2))
            out[variant]["peak_allocated_gib"].append(round(torch.cuda.max_memory_allocated() / 2**30, 3))
            del st
            gc.collect()
            torch.cuda.empty_cache()
    return {"size": [B, n, d], **out}


MEASUREMENTS = tuple(f"pgpe_{n}" for n in SPECS) + tuple(f"pgpe_{n}_vs_torch" for n in SPECS) + (
    "pgpe_input_noise_sphere_lazy", "functional_input_noise_sphere")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pgpe", type=int, nargs=2, default=[1_000_000, 10_000])
    ap.add_argument("--torch-pgpe", type=int, nargs=2, default=[200_000, 10_000])
    ap.add_argument("--lazy-pgpe", type=int, nargs=2, default=[1_000_000, 100_000])
    ap.add_argument("--lazy-gens", type=int, default=3)
    ap.add_argument("--functional", type=int, nargs=3, default=[1024, 1000, 1000])
    ap.add_argument("--only", nargs="+", choices=MEASUREMENTS, default=list(MEASUREMENTS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("noisy_objective_bench.py measures on a GPU: none found")
    noisy = {n: FusedObjective(f"noisy_{n}", **kw) for n, (kw, _) in SPECS.items()}
    twins = {n: FusedObjective(f"twin_{n}", **kw) for n, (_, kw) in SPECS.items()}
    for o in noisy.values():
        o.compile_batched()
    res = {"card": card(), "gens": args.gens, "rounds": args.rounds,
           "kernels": {o.name: {"registers": sorted({i["registers"] for i in o.kernel_info.values()}),
                                "batched_registers": sorted({i["registers"] for i in o.batched_kernel_info.values()}),
                                "spill_bytes": sum(i["spill_stores"] + i["spill_loads"] for info in (o.kernel_info, o.batched_kernel_info)
                                                   for i in info.values())} for o in noisy.values()}}
    print(json.dumps({"card": res["card"], "kernels": res["kernels"]}), file=sys.stderr, flush=True)
    run = {}
    for n in SPECS:
        run[f"pgpe_{n}"] = lambda n=n: pair(pgpe, ("noisy", noisy[n]), ("twin", twins[n]), *args.pgpe, args)
        run[f"pgpe_{n}_vs_torch"] = lambda n=n: pair(pgpe, ("fused", noisy[n]), ("torch", TORCH[n]), *args.torch_pgpe, args)
    run["pgpe_input_noise_sphere_lazy"] = lambda: lazy_pair(("noisy", noisy["input_noise_sphere"]), ("twin", twins["input_noise_sphere"]),
                                                            *args.lazy_pgpe, args)
    run["functional_input_noise_sphere"] = lambda: functional(*args.functional, noisy["input_noise_sphere"], TORCH["input_noise_sphere"], args)
    for name in MEASUREMENTS:
        if name in args.only:
            res[name] = run[name]()
            print(json.dumps({name: res[name]}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
