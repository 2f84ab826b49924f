"""Seconds per generation of separable CMA-ES (`CMAES(..., separable=True)`, Rastrigin, CUDA float32):
python scripts/sepcma_bench.py [--cmp N D] [--big N D] [--gens K] [--warmup W] [--rounds R]

At the comparison size (default 100 000 x 4 096) three searchers run from the same seed: the fused generation with a
materialised population, the fused generation with a lazy one, and the op-by-op path (the mirror of the reference's `_step`).
At the large size (default 1 000 000 x 10 000) only the two fused ones run: the op-by-op path's N x D temporaries do not fit.
Every searcher first takes W warm-up generations (its peak memory, `torch.cuda.max_memory_allocated` above what was allocated
before it was built, is read then); the timed windows of K generations then alternate between the searchers of a size, R
rounds, each window timed with CUDA events around the steps and ended by a device synchronise.  Before any speed-up is
quoted the final m, sigma and C of the fused and op-by-op runs at the comparison size are compared (same seed, same number of
generations, same Philox draws).  A last, separate window per fused searcher records the per-kernel CUDA-event timers.
The card name and power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from evotorch_b200 import Problem, ops  # noqa: E402
from evotorch_b200.algorithms import CMAES  # noqa: E402
from evotorch_b200.objectives import rastrigin  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ("?", "?", "?")
    return {"name": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power, "max_sm_clock": clock}


def build(n: int, d: int, mode: str, warmup: int):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=d, device="cuda", seed=7, lazy_population=mode == "lazy")
    # an explicit centre: with center_init=None a materialised searcher draws its initial population before its random centre
    center = torch.rand(d, generator=torch.Generator().manual_seed(d), dtype=torch.float32) * 10.24 - 5.12
    s = CMAES(prob, stdev_init=1.0, popsize=n, separable=True, center_init=center.cuda())
    if mode == "op_by_op":
        s._fused_ok = lambda: False
    for _ in range(warmup):
        s.step()
    torch.cuda.synchronize()
    return s, (torch.cuda.max_memory_allocated() - base) / 2**20


def window(s, gens: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(gens):
        s.step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / gens


def kernel_times(s, gens: int) -> dict:
    ops.enable_timers()
    for _ in range(gens):
        s.step()
    torch.cuda.synchronize()
    res = {k: round(ms, 4) for k, (cnt, ms) in ops.timer_results().items()}
    ops.disable_timers()
    return res


def rel_diff(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def run_size(n: int, d: int, modes, gens: int, warmup: int, rounds: int) -> dict:
    searchers, out = {}, {"popsize": n, "dim": d, "peak_mib": {}, "ms_per_gen": {m: [] for m in modes}}
    for m in modes:
        searchers[m], out["peak_mib"][m] = build(n, d, m, warmup)
        out["peak_mib"][m] = round(out["peak_mib"][m], 1)
    for _ in range(rounds):
        for m in modes:
            out["ms_per_gen"][m].append(round(window(searchers[m], gens), 3))
    # every searcher has now taken the same number of generations from the same seed
    if "op_by_op" in searchers:
        f, r = searchers["fused"], searchers["op_by_op"]
        out["fused_vs_op_by_op_rel_diff"] = {"m": rel_diff(f.m, r.m), "sigma": rel_diff(f.sigma, r.sigma), "C": rel_diff(f.C, r.C)}
    if "lazy" in searchers and "fused" in searchers:
        f, z = searchers["fused"], searchers["lazy"]
        out["lazy_equals_fused"] = all(torch.equal(getattr(f, k), getattr(z, k)) for k in ("m", "sigma", "C", "A", "p_sigma", "p_c"))
    out["kernel_ms"] = {m: kernel_times(searchers[m], gens) for m in modes if m != "op_by_op"}
    del searchers
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cmp", type=int, nargs=2, default=[100_000, 4096])
    ap.add_argument("--big", type=int, nargs=2, default=[1_000_000, 10_000])
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sepcma_bench.py measures the GPU path and needs a CUDA device")
    res = {"card": card(), "gens_per_window": args.gens, "warmup": args.warmup, "rounds": args.rounds}
    res["comparison"] = run_size(*args.cmp, ("fused", "lazy", "op_by_op"), args.gens, args.warmup, args.rounds)
    res["large"] = run_size(*args.big, ("fused", "lazy"), args.gens, args.warmup, args.rounds)
    res["card_after"] = card()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
