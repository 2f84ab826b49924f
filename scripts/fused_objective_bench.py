"""Generations per second of user-defined objectives fused into the sampler (`objectives.FusedObjective`), against the built-in
objectives and against the same function as a plain torch callable (sample, then evaluate with torch):

python scripts/fused_objective_bench.py [--gens K] [--warmup W] [--rounds R] [--pgpe N D] [--torch-pgpe N D] [--sep N D]

PGPE (symmetric, ClipUp) pairs:
  - built-in sphere     vs the FusedObjective sphere twin                    at --pgpe (default 1 000 000 x 10 000)
  - built-in rastrigin  vs the FusedObjective Rastrigin twin (precise cosf)  at --pgpe
  - Styblinski-Tang fused vs the same formula as a torch callable            at --torch-pgpe (default 200 000 x 10 000: the torch
    expression's N x D temporaries do not fit next to a 1 M x 10 k population)
Separable CMA-ES: Styblinski-Tang fused vs torch callable at --sep (default 100 000 x 4 096).
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pgpe", type=int, nargs=2, default=[1_000_000, 10_000])
    ap.add_argument("--torch-pgpe", type=int, nargs=2, default=[200_000, 10_000])
    ap.add_argument("--sep", type=int, nargs=2, default=[100_000, 4_096])
    args = ap.parse_args()
    twin = FusedObjective("sphere_twin", {"s": "x**2"}, "s")
    rastrigin_twin = FusedObjective("rastrigin_twin", {"a": "x**2", "c": "cos(2*pi*x)"}, "10*D + a - 10*c")
    st = FusedObjective("styblinski_tang", {"s": "x**4 - 16*x**2 + 5*x"}, "0.5 * s")
    res = {"card": card(), "gens": args.gens, "rounds": args.rounds,
           "registers": {o.name: max(i["registers"] for e, i in o.kernel_info.items() if "sample_eval_kernel" in e) for o in (twin, rastrigin_twin, st)}}
    res["pgpe_sphere"] = pair(pgpe, ("builtin", sphere), ("fused", twin), *args.pgpe, args)
    res["pgpe_rastrigin"] = pair(pgpe, ("builtin", rastrigin), ("fused", rastrigin_twin), *args.pgpe, args)
    res["pgpe_styblinski_tang"] = pair(pgpe, ("fused", st), ("torch", torch_styblinski_tang), *args.torch_pgpe, args)
    res["sepcma_styblinski_tang"] = pair(sep, ("fused", st), ("torch", torch_styblinski_tang), *args.sep, args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
