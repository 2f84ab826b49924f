"""Generations per second of user-defined objectives fused into the sampler (`objectives.FusedObjective`), against the built-in
objectives and against the same function as a plain torch callable (sample, then evaluate with torch):

python scripts/fused_objective_bench.py [--gens K] [--warmup W] [--rounds R] [--pgpe N D] [--torch-pgpe N D] [--sep N D]
                                        [--lazy-pgpe N D] [--lazy-gens K] [--only NAME ...]

PGPE (symmetric, ClipUp) pairs:
  - built-in sphere     vs the FusedObjective sphere twin                    at --pgpe (default 1 000 000 x 10 000)
  - built-in rastrigin  vs the FusedObjective Rastrigin twin (precise cosf)  at --pgpe
  - Styblinski-Tang fused vs the same formula as a torch callable            at --torch-pgpe (default 200 000 x 10 000: the torch
    expression's N x D temporaries do not fit next to a 1 M x 10 k population)
Separable CMA-ES: Styblinski-Tang fused vs torch callable at --sep (default 100 000 x 4 096).
Rosenbrock, a FusedObjective with a pair term (x_j and x_{j+1}):
  - PGPE: fused Rosenbrock vs the fused sphere twin at --pgpe (the cost of the neighbour term), and vs the same formula as a
    torch callable at --torch-pgpe;
  - separable CMA-ES: fused vs torch callable at --sep;
  - PGPE with the lazy population at --lazy-pgpe (default 1 000 000 x 100 000; no torch callable can run this size): generations
    per second over --lazy-gens generations and the peak allocated memory.
--only runs a subset of the measurements by name (default: all).
The timed windows of K generations alternate between the two variants of a pair, R rounds; each window builds its searcher,
takes W warm-up generations, then times K with CUDA events and ends with a synchronise.  The sampler kernel time is the mean of the library's
CUDA-event timers ("sample_eval" for the fused kernel, "sample" for the sample-only one) over one more window.  The card name and
power limit are read in the same run.  Prints one JSON line."""
import argparse
import gc
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from evotorch_b200 import Problem, ops  # noqa: E402
from evotorch_b200.algorithms import CMAES, PGPE  # noqa: E402
from evotorch_b200.objectives import FusedObjective, rastrigin, sphere  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?", "?"])[:2] if q.returncode == 0 else ("?", "?")
    return {"name": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def torch_styblinski_tang(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * torch.sum(x**4 - 16 * x**2 + 5 * x, dim=-1)


torch_styblinski_tang.__evotorch_vectorized__ = True


def torch_rosenbrock(x: torch.Tensor) -> torch.Tensor:
    return torch.sum(100 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1 - x[..., :-1]) ** 2, dim=-1)


torch_rosenbrock.__evotorch_vectorized__ = True


def pgpe(objective, n: int, d: int):
    prob = Problem("min", objective, initial_bounds=(-5, 5), solution_length=d, device="cuda", seed=1)
    return PGPE(prob, popsize=n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)


def sep(objective, n: int, d: int):
    prob = Problem("min", objective, initial_bounds=(-5, 5), solution_length=d, device="cuda", seed=1)
    return CMAES(prob, stdev_init=1.0, popsize=n, separable=True)


def window(s, k: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(k):
        s.step()
    b.record()
    torch.cuda.synchronize()
    return k / (a.elapsed_time(b) / 1e3)


def sampler_ms(s, k: int) -> dict:
    ops.enable_timers()
    for _ in range(k):
        s.step()
    torch.cuda.synchronize()
    res = {name: round(ms, 3) for name, (_, ms) in ops.timer_results().items() if name in ("sample_eval", "sample", "sepcma_sample")}
    ops.disable_timers()
    return res


def pair(make, a, b, n: int, d: int, args) -> dict:
    """Alternating windows; each window builds its searcher afresh (two 1 M x 10 k populations do not fit on one card together)."""
    out = {label: {"gens_per_s": []} for label, _ in (a, b)}
    for r in range(args.rounds):
        for label, objective in (a, b):
            s = make(objective, n, d)
            for _ in range(args.warmup):
                s.step()
            out[label]["gens_per_s"].append(round(window(s, args.gens), 3))
            if r == args.rounds - 1:
                out[label]["sampler_ms"] = sampler_ms(s, args.gens)
            del s
            gc.collect()  # searchers hold reference cycles: free the population before the next one is built
            torch.cuda.empty_cache()
    return {"size": [n, d], **out}


def lazy(objective, n: int, d: int, args) -> dict:
    """PGPE with the lazy population (no N x D matrix): generations per second and the peak allocated memory."""
    prob = Problem("min", objective, initial_bounds=(-5, 5), solution_length=d, device="cuda", seed=1, lazy_population=True)
    s = PGPE(prob, popsize=n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    for _ in range(args.warmup):
        s.step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    rates = [round(window(s, args.lazy_gens), 3) for _ in range(args.rounds)]
    peak = torch.cuda.max_memory_allocated() / 2**30
    out = {"size": [n, d], "gens_per_s": rates, "peak_allocated_gib": round(peak, 3), "sampler_ms": sampler_ms(s, args.lazy_gens)}
    del s
    gc.collect()
    torch.cuda.empty_cache()
    return out


MEASUREMENTS = ("pgpe_sphere", "pgpe_rastrigin", "pgpe_styblinski_tang", "sepcma_styblinski_tang", "pgpe_rosenbrock_vs_sphere",
                "pgpe_rosenbrock", "sepcma_rosenbrock", "pgpe_rosenbrock_lazy")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pgpe", type=int, nargs=2, default=[1_000_000, 10_000])
    ap.add_argument("--torch-pgpe", type=int, nargs=2, default=[200_000, 10_000])
    ap.add_argument("--sep", type=int, nargs=2, default=[100_000, 4_096])
    ap.add_argument("--lazy-pgpe", type=int, nargs=2, default=[1_000_000, 100_000])
    ap.add_argument("--lazy-gens", type=int, default=3)
    ap.add_argument("--only", nargs="+", choices=MEASUREMENTS, default=list(MEASUREMENTS))
    args = ap.parse_args()
    twin = FusedObjective("sphere_twin", {"s": "x**2"}, "s")
    rastrigin_twin = FusedObjective("rastrigin_twin", {"a": "x**2", "c": "cos(2*pi*x)"}, "10*D + a - 10*c")
    st = FusedObjective("styblinski_tang", {"s": "x**4 - 16*x**2 + 5*x"}, "0.5 * s")
    rosen = FusedObjective("rosenbrock", {"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s")
    res = {"card": card(), "gens": args.gens, "rounds": args.rounds,
           "registers": {o.name: max(i["registers"] for e, i in o.kernel_info.items() if "sample_eval_kernel" in e)
                         for o in (twin, rastrigin_twin, st, rosen)}}
    run = {
        "pgpe_sphere": lambda: pair(pgpe, ("builtin", sphere), ("fused", twin), *args.pgpe, args),
        "pgpe_rastrigin": lambda: pair(pgpe, ("builtin", rastrigin), ("fused", rastrigin_twin), *args.pgpe, args),
        "pgpe_styblinski_tang": lambda: pair(pgpe, ("fused", st), ("torch", torch_styblinski_tang), *args.torch_pgpe, args),
        "sepcma_styblinski_tang": lambda: pair(sep, ("fused", st), ("torch", torch_styblinski_tang), *args.sep, args),
        "pgpe_rosenbrock_vs_sphere": lambda: pair(pgpe, ("fused_rosenbrock", rosen), ("fused_sphere_twin", twin), *args.pgpe, args),
        "pgpe_rosenbrock": lambda: pair(pgpe, ("fused", rosen), ("torch", torch_rosenbrock), *args.torch_pgpe, args),
        "sepcma_rosenbrock": lambda: pair(sep, ("fused", rosen), ("torch", torch_rosenbrock), *args.sep, args),
        "pgpe_rosenbrock_lazy": lambda: lazy(rosen, *args.lazy_pgpe, args),
    }
    for name in MEASUREMENTS:
        if name in args.only:
            res[name] = run[name]()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
