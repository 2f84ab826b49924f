"""Functional PGPE / CEM on batches of searches: one generation (ask, evaluate, tell) with the objective evaluated four ways.

    (a) `*_ask` + the objective's torch expression on the (B, N, D) population + tell
    (b) `*_ask` + `ops.evaluate` (the stand-alone K2 kernel) on the flattened (B*N, D) rows + tell
    (c) `*_ask_and_evaluate`: sampled and evaluated in one launch, population stored + tell
    (d) `*_ask_and_evaluate(lazy=True)`: nothing stored, the tell rebuilds the rows it needs

Objectives: Rastrigin (built-in) and Rosenbrock (a FusedObjective with a pair term).  Shapes B x N x D: 1024 x 1000 x 1000,
64 x 10 000 x 1000 and 10 000 x 100 x 100.  Reported per workload and variant: milliseconds per generation (CUDA events over a
window of generations, the median of alternating windows) and the peak memory allocated during a window above what was allocated
before it.  Also the time of a plain `pgpe_ask` (the sample-only batched sampler) and of its sampling call alone
(evok_sample_batched through ctypes), on this libevok.so and, with --parent-lib, on an older one with the same Python code, in
alternating windows.  The card's name and enforced power limit are read in the same run.

    python scripts/functional_fused_bench.py [--gens 5] [--windows 3] [--parent-lib path/to/libevok.so] [--out file.json]
"""

import argparse
import contextlib
import ctypes
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evotorch_b200 import _native as nat  # noqa: E402
from evotorch_b200 import ops  # noqa: E402
from evotorch_b200.algorithms import functional as F  # noqa: E402
from evotorch_b200.algorithms.functional.misc import draw_philox_seed  # noqa: E402
from evotorch_b200.objectives import FusedObjective, rastrigin  # noqa: E402

SHAPES = [(1024, 1000, 1000), (64, 10_000, 1000), (10_000, 100, 100)]
VARIANTS = ["a_torch", "b_evaluate", "c_fused", "d_lazy"]


def make_state(algo, B, D):
    center = torch.zeros(B, D, device="cuda") + 0.5
    if algo == "pgpe":
        return F.pgpe(center_init=center, center_learning_rate=0.1, stdev_learning_rate=0.1, stdev_init=1.0, objective_sense="min")
    return F.cem(center_init=center, stdev_init=1.0, parenthood_ratio=0.25, objective_sense="min", stdev_max_change=0.2)


def generation(algo, variant, obj, state, N):
    ask = F.pgpe_ask if algo == "pgpe" else F.cem_ask
    ask_eval = F.pgpe_ask_and_evaluate if algo == "pgpe" else F.cem_ask_and_evaluate
    tell = F.pgpe_tell if algo == "pgpe" else F.cem_tell
    if variant == "a_torch":
        values = ask(state, popsize=N)
        evals = obj._torch_fn(values)
    elif variant == "b_evaluate":
        values = ask(state, popsize=N)
        evals = ops.evaluate(obj.evok_objective_id, values.view(-1, values.shape[-1])).view(values.shape[:-1])
    else:
        values, evals = ask_eval(state, popsize=N, objective=obj, lazy=(variant == "d_lazy"))
    return tell(state, values, evals)


def window(fn, gens):
    """(ms per call, peak bytes allocated above the start) of `gens` calls of fn after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(gens):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / gens, torch.cuda.max_memory_allocated() - base


def sampler(path=None):
    lib = nat.lib() if path is None else ctypes.CDLL(path)
    fn = lib.evok_sample_batched
    fn.restype = ctypes.c_int
    fn.argtypes = nat._SIGNATURES["evok_sample_batched"][1]
    return fn


@contextlib.contextmanager
def library(path):
    """Inside the block the package calls the libevok.so at `path` (its evok_sample_batched: the only kernel pgpe_ask launches)."""
    handle = ctypes.CDLL(path)
    for name in ("evok_sample_batched", "evok_error_string"):
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = nat._SIGNATURES[name]
    saved, nat._lib = nat.lib(), handle
    try:
        yield
    finally:
        nat._lib = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--shapes", default="all")
    ap.add_argument("--out", default=None)
    ap.add_argument("--ask-only", action="store_true", help="time only pgpe_ask and its sampling call")
    args = ap.parse_args()
    torch.manual_seed(0)
    power = nat.lib().evok_grad_power_limit_mw(torch.cuda.current_device())
    result = {"device": torch.cuda.get_device_name(), "power_limit_w": power / 1000 if power > 0 else None, "gens_per_window": args.gens,
              "windows": args.windows, "workloads": [], "pgpe_ask": []}
    rosenbrock = FusedObjective("rosenbrock", {"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s")
    rosenbrock.compile_batched()
    shapes = SHAPES if args.shapes == "all" else [SHAPES[int(i)] for i in args.shapes.split(",")]
    libs = {"sample_batched": sampler()}
    if args.parent_lib:
        libs["sample_batched_parent_lib"] = sampler(args.parent_lib)
    for B, N, D in shapes:
        # plain pgpe_ask, and the same sampling call on the parent library, alternating
        state = make_state("pgpe", B, D)
        out = torch.empty(B, N, D, device="cuda")
        center, stdev = state.optimizer_state.center, state.stdev
        times = {"pgpe_ask": [], **({"pgpe_ask_parent_lib": []} if args.parent_lib else {}), **{k: [] for k in libs}}
        for _ in range(args.windows):
            times["pgpe_ask"].append(window(lambda: F.pgpe_ask(state, popsize=N), args.gens)[0])
            if args.parent_lib:
                with library(args.parent_lib):
                    times["pgpe_ask_parent_lib"].append(window(lambda: F.pgpe_ask(state, popsize=N), args.gens)[0])
            for k, fn in libs.items():
                def call(fn=fn):
                    nat.check(fn(out.data_ptr(), N * D, D, center.data_ptr(), D, stdev.data_ptr(), 0, B, N, D, 1, draw_philox_seed(), 0,
                                 nat.stream_of(out)), "evok_sample_batched")
                times[k].append(window(call, args.gens)[0])
        del out
        result["pgpe_ask"].append({"shape": [B, N, D], **{k: statistics.median(v) for k, v in times.items()}, "windows_ms": times})
        print(json.dumps(result["pgpe_ask"][-1]), flush=True)
        if args.ask_only:
            continue
        for algo in ("pgpe", "cem"):
            for name, obj in (("rastrigin", rastrigin), ("rosenbrock", rosenbrock)):
                rows = {v: [] for v in VARIANTS}
                peaks = {}
                for _ in range(args.windows):
                    for v in VARIANTS:
                        holder = {"s": make_state(algo, B, D)}

                        def step():
                            holder["s"] = generation(algo, v, obj, holder["s"], N)
                        ms, peak = window(step, args.gens)
                        rows[v].append(ms)
                        peaks[v] = max(peaks.get(v, 0), peak)
                        del holder
                        torch.cuda.empty_cache()
                entry = {"algo": algo, "objective": name, "shape": [B, N, D],
                         "ms_per_generation": {v: statistics.median(t) for v, t in rows.items()},
                         "peak_allocated_gb": {v: p / 1e9 for v, p in peaks.items()}, "windows_ms": rows}
                result["workloads"].append(entry)
                print(json.dumps(entry), flush=True)
    print(json.dumps({k: result[k] for k in ("device", "power_limit_w", "pgpe_ask")}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
