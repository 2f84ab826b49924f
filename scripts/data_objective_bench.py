"""What the data of a FusedObjective costs, and what it buys over a torch callable:

python scripts/data_objective_bench.py [--gens K] [--warmup W] [--rounds R] [--pgpe N D] [--torch-pgpe N D] [--lazy-pgpe N D]
                                       [--lazy-gens K] [--functional B N D ...] [--only NAME ...]

PGPE (symmetric, ClipUp) at --pgpe (default 1 000 000 x 10 000), each against its twin without data (the cost of the loads):
  - shifted sphere (x - o)**2                      vs the fused sphere x**2              (one vector)
  - weighted least squares w * (x - t)**2 + lam*D  vs the fused sphere                   (two vectors and a scalar)
  - shifted Rosenbrock                             vs the fused Rosenbrock               (one vector in a pair term)
Least squares fused vs the same function as a torch callable at --torch-pgpe (default 200 000 x 10 000).
The shifted sphere on the lazy population at --lazy-pgpe (default 1 000 000 x 100 000), with the peak allocated memory.
Functional PGPE with one target per batch item at --functional (default 1024 x 1000 x 1000 and 64 x 10 000 x 1000): the fused
sampler with a stored and with a lazy population against `pgpe_ask` followed by the torch expression, with the peak memory.
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
from fused_objective_bench import card, lazy, pair, pgpe  # noqa: E402

from evotorch_b200.algorithms.functional import pgpe as func_pgpe  # noqa: E402
from evotorch_b200.algorithms.functional import pgpe_ask, pgpe_ask_and_evaluate, pgpe_tell  # noqa: E402
from evotorch_b200.objectives import FusedObjective  # noqa: E402


def functional(B: int, n: int, d: int, args) -> dict:
    """Generations per second and peak allocated GiB of functional PGPE on B searches, item b minimising |x - target_b|^2."""
    targets = torch.randn(B, d, device="cuda")
    fused = FusedObjective("shifted_sphere", {"s": "(x - o)**2"}, "s", data={"o": targets})

    def torch_expr(x):
        return ((x - targets[:, None, :]) ** 2).sum(-1)

    def generation(st, variant):
        if variant == "torch":
            values = pgpe_ask(st, popsize=n)
            evals = torch_expr(values)
        else:
            values, evals = pgpe_ask_and_evaluate(st, popsize=n, objective=fused, lazy=variant == "fused_lazy")
        return pgpe_tell(st, values, evals)

    out = {v: {"gens_per_s": []} for v in ("fused_stored", "fused_lazy", "torch")}
    for r in range(args.rounds):
        for variant in out:
            st = func_pgpe(center_init=torch.zeros(B, d, device="cuda"), center_learning_rate=0.3, stdev_learning_rate=0.1,
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


MEASUREMENTS = ("pgpe_shifted_sphere", "pgpe_least_squares", "pgpe_shifted_rosenbrock", "pgpe_least_squares_vs_torch",
                "pgpe_shifted_sphere_lazy", "functional")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pgpe", type=int, nargs=2, default=[1_000_000, 10_000])
    ap.add_argument("--torch-pgpe", type=int, nargs=2, default=[200_000, 10_000])
    ap.add_argument("--lazy-pgpe", type=int, nargs=2, default=[1_000_000, 100_000])
    ap.add_argument("--lazy-gens", type=int, default=3)
    ap.add_argument("--functional", type=int, nargs="+", default=[1024, 1000, 1000, 64, 10_000, 1000])
    ap.add_argument("--only", nargs="+", choices=MEASUREMENTS, default=list(MEASUREMENTS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("data_objective_bench.py measures on a GPU: none found")
    if len(args.functional) % 3:
        ap.error("--functional takes B N D triples")
    d, dt, dl = args.pgpe[1], args.torch_pgpe[1], args.lazy_pgpe[1]

    def vec(n, positive=False):
        t = torch.randn(n, device="cuda")
        return t.abs() + 0.1 if positive else t

    sums_lsq, value_lsq = {"s": "w * (x - t)**2"}, "s + lam * D"
    lam = torch.tensor([0.1], device="cuda")
    twin = FusedObjective("sphere_twin", {"s": "x**2"}, "s")
    rosen = FusedObjective("rosenbrock", {"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s")
    shifted = FusedObjective("shifted_sphere", {"s": "(x - o)**2"}, "s", data={"o": vec(d)})
    lsq = FusedObjective("least_squares", sums_lsq, value_lsq, data={"t": vec(d), "w": vec(d, True), "lam": lam})
    srosen = FusedObjective("shifted_rosenbrock", {"s": "100*((xn - o_n) - (x - o)**2)**2 + (1 - (x - o))**2"}, "s", data={"o": vec(d)})
    tt, tw = vec(dt), vec(dt, True)
    lsq_t = lsq.with_data(t=tt, w=tw, lam=lam)

    def torch_lsq(x):
        return torch.sum(tw * (x - tt) ** 2, dim=-1) + 0.1 * x.shape[-1]

    torch_lsq.__evotorch_vectorized__ = True
    for o in (shifted, lsq, srosen):
        o.compile_batched()
    res = {"card": card(), "gens": args.gens, "rounds": args.rounds,
           "kernels": {o.name: {"max_registers": max(i["registers"] for info in (o.kernel_info, o.batched_kernel_info) for i in info.values()),
                                "spill_bytes": sum(i["spill_stores"] + i["spill_loads"] for info in (o.kernel_info, o.batched_kernel_info)
                                                   for i in info.values())} for o in (shifted, lsq, srosen)}}
    run = {
        "pgpe_shifted_sphere": lambda: pair(pgpe, ("shifted_sphere", shifted), ("sphere_twin", twin), *args.pgpe, args),
        "pgpe_least_squares": lambda: pair(pgpe, ("least_squares", lsq), ("sphere_twin", twin), *args.pgpe, args),
        "pgpe_shifted_rosenbrock": lambda: pair(pgpe, ("shifted_rosenbrock", srosen), ("rosenbrock", rosen), *args.pgpe, args),
        "pgpe_least_squares_vs_torch": lambda: pair(pgpe, ("fused", lsq_t), ("torch", torch_lsq), *args.torch_pgpe, args),
        "pgpe_shifted_sphere_lazy": lambda: lazy(shifted.with_data(o=vec(dl)), *args.lazy_pgpe, args),
        "functional": lambda: [functional(*args.functional[i:i + 3], args) for i in range(0, len(args.functional), 3)],
    }
    for name in MEASUREMENTS:
        if name in args.only:
            res[name] = run[name]()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
