"""What products, maxima, running sums and conditionals in a FusedObjective cost, and what they buy over a torch callable:

python scripts/reduction_objective_bench.py [--gens K] [--warmup W] [--rounds R] [--pgpe N D] [--torch-pgpe N D] [--lazy-pgpe N D]
                                            [--lazy-gens K] [--sep N D] [--functional B N D] [--only NAME ...]

PGPE (symmetric, ClipUp) at --pgpe (default 1 000 000 x 10 000), each against the fused x**2 sphere twin (the cost of the combine
operations and of the running-sum scan over a plain sum):
  - Griewank        1 + sum x^2 / 4000 - prod cos(x_j / sqrt(j + 1))     (a product)
  - Schwefel 2.22   sum |x| + prod |x|                                  (a product)
  - Schwefel 2.21   max |x|                                             (a maximum)
  - Schwefel 1.2    sum_j (sum_{k<=j} x_k)^2                            (a running sum)
The same four fused against the same functions as torch callables at --torch-pgpe (default 200 000 x 10 000).
Schwefel 1.2 on the lazy population at --lazy-pgpe (default 1 000 000 x 100 000), with the peak allocated memory.
Separable CMA-ES on Schwefel 1.2 at --sep (default 100 000 x 4096), fused against the torch callable.
Functional PGPE with Griewank at --functional (default 1024 x 1000 x 1000): the fused sampler with a stored and with a lazy
population against `pgpe_ask` followed by the torch expression, with the peak memory.
The windows of a pair alternate, R rounds, each after W warm-up generations, timed with CUDA events and ended by a synchronise
(scripts/fused_objective_bench.py has the window functions).  Needs a GPU; prints the card and its power limit with one JSON line."""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fused_objective_bench import card, lazy, pair, pgpe, sep  # noqa: E402

from evotorch_b200.algorithms.functional import pgpe as func_pgpe  # noqa: E402
from evotorch_b200.algorithms.functional import pgpe_ask, pgpe_ask_and_evaluate, pgpe_tell  # noqa: E402
from evotorch_b200.objectives import FusedObjective  # noqa: E402

SPECS = {
    "griewank": dict(sums={"s": "x**2"}, prods={"p": "cos(x / sqrt(j + 1))"}, value="1 + s / 4000 - p"),
    "schwefel_2_22": dict(sums={"a": "abs(x)"}, prods={"p": "abs(x)"}, value="a + p"),
    "schwefel_2_21": dict(maxs={"m": "abs(x)"}, value="m"),
    "schwefel_1_2": dict(running={"c": "x"}, sums={"s": "c**2"}, value="s"),
}


def _vectorized(fn):
    fn.__evotorch_vectorized__ = True
    return fn


TORCH = {
    "griewank": _vectorized(lambda x: 1 + (x**2).sum(-1) / 4000
                            - torch.cos(x / torch.sqrt(torch.arange(1, x.shape[-1] + 1, device=x.device, dtype=x.dtype))).prod(-1)),
    "schwefel_2_22": _vectorized(lambda x: x.abs().sum(-1) + x.abs().prod(-1)),
    "schwefel_2_21": _vectorized(lambda x: x.abs().amax(-1)),
    "schwefel_1_2": _vectorized(lambda x: (x.cumsum(-1) ** 2).sum(-1)),
}


def make(name):
    kw = dict(SPECS[name])
    return FusedObjective(name, kw.pop("sums", None), kw.pop("value"), **kw)


def functional(B: int, n: int, d: int, args) -> dict:
    """Generations per second and peak allocated GiB of functional PGPE on B Griewank searches."""
    fused = make("griewank")
    fused.compile_batched()

    def generation(st, variant):
        if variant == "torch":
            values = pgpe_ask(st, popsize=n)
            evals = TORCH["griewank"](values)
        else:
            values, evals = pgpe_ask_and_evaluate(st, popsize=n, objective=fused, lazy=variant == "fused_lazy")
        return pgpe_tell(st, values, evals)

    out = {v: {"gens_per_s": []} for v in ("fused_stored", "fused_lazy", "torch")}
    for r in range(args.rounds):
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
            out[variant]["peak_allocated_gib"] = round(torch.cuda.max_memory_allocated() / 2**30, 3)
            del st
            gc.collect()
            torch.cuda.empty_cache()
    return {"size": [B, n, d], **out}


MEASUREMENTS = tuple(f"pgpe_{n}" for n in SPECS) + tuple(f"pgpe_{n}_vs_torch" for n in SPECS) + (
    "pgpe_schwefel_1_2_lazy", "sepcma_schwefel_1_2_vs_torch", "functional_griewank")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pgpe", type=int, nargs=2, default=[1_000_000, 10_000])
    ap.add_argument("--torch-pgpe", type=int, nargs=2, default=[200_000, 10_000])
    ap.add_argument("--lazy-pgpe", type=int, nargs=2, default=[1_000_000, 100_000])
    ap.add_argument("--lazy-gens", type=int, default=3)
    ap.add_argument("--sep", type=int, nargs=2, default=[100_000, 4096])
    ap.add_argument("--functional", type=int, nargs=3, default=[1024, 1000, 1000])
    ap.add_argument("--only", nargs="+", choices=MEASUREMENTS, default=list(MEASUREMENTS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("reduction_objective_bench.py measures on a GPU: none found")
    twin = FusedObjective("sphere_twin", {"s": "x**2"}, "s")
    objs = {name: make(name) for name in SPECS}
    for o in objs.values():
        o.compile_batched()
    res = {"card": card(), "gens": args.gens, "rounds": args.rounds,
           "kernels": {o.name: {"registers": sorted({i["registers"] for i in o.kernel_info.values()}),
                                "batched_registers": sorted({i["registers"] for i in o.batched_kernel_info.values()}),
                                "spill_bytes": sum(i["spill_stores"] + i["spill_loads"] for info in (o.kernel_info, o.batched_kernel_info)
                                                   for i in info.values())} for o in objs.values()}}
    run = {}
    for name, o in objs.items():
        run[f"pgpe_{name}"] = lambda o=o, name=name: pair(pgpe, (name, o), ("sphere_twin", twin), *args.pgpe, args)
        run[f"pgpe_{name}_vs_torch"] = lambda o=o, name=name: pair(pgpe, ("fused", o), ("torch", TORCH[name]), *args.torch_pgpe, args)
    run["pgpe_schwefel_1_2_lazy"] = lambda: lazy(objs["schwefel_1_2"], *args.lazy_pgpe, args)
    run["sepcma_schwefel_1_2_vs_torch"] = lambda: pair(sep, ("fused", objs["schwefel_1_2"]), ("torch", TORCH["schwefel_1_2"]), *args.sep, args)
    run["functional_griewank"] = lambda: functional(*args.functional, args)
    for name in MEASUREMENTS:
        if name in args.only:
            res[name] = run[name]()
            print(json.dumps({name: res[name]}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
