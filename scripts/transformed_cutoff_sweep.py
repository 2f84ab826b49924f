"""Where the fused path of the transformed evaluation stops paying: both paths timed at the same D on the H100.

    python scripts/transformed_cutoff_sweep.py --build          (where nvcc is: the two builds below, into evotorch_b200/lib/)
    python scripts/transformed_cutoff_sweep.py [--rounds 3] [--windows 5] [--out FILE]      (on the GPU)

`evok_eval_transform_batched` chooses its path from D alone, at the build-time cutoff EVOK_TRANSFORM_FUSED_MAX_D.  Two builds
fix the choice: libevok_tfgemm.so (cutoff 0: the GEMM path at every D) and libevok_tffused.so (cutoff 236: the fused path up to
the 227 KB of shared memory a CTA can take).  Each build runs in a process of its own (the objective registers with the library it
loaded); the processes alternate, `--rounds` times each.  Workload: rotated Rastrigin with a per-item rotation M_b and offset o_b,
B items of n = 4 + floor(3 ln D) rows (CMA-ES's default population size) at B = 64 and 1024, D from 8 to 236; CUDA events around
windows of calls, median over the windows of every round, then the median over the rounds.  The card's name and power limit are
read in the same run.  One JSON object is printed (and written to --out).
"""

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {"gemm": ("tfgemm", "EVOK_TRANSFORM_FUSED_MAX_D=0"), "fused": ("tffused", "EVOK_TRANSFORM_FUSED_MAX_D=236")}
DIMS = [8, 16, 32, 48, 64, 80, 96, 112, 128, 144, 160, 192, 224, 236]
ITEMS = [64, 1024]


def popsize(D: int) -> int:
    return 4 + int(3 * math.log(D))


def worker(lib_path: str, windows: int) -> dict:
    """Median ms per call of every (B, D) with the library at lib_path."""
    from evotorch_b200 import _native as nat

    nat.LIB_PATH = lib_path  # before the first load: every kernel of this process comes from this build
    import torch

    from evotorch_b200.objectives import FusedObjective

    dev = torch.device("cuda")
    out = {}
    for B in ITEMS:
        for D in DIMS:
            g = torch.Generator(device=dev).manual_seed(D)
            M = torch.linalg.qr(torch.randn(B, D, D, device=dev, generator=g))[0].contiguous()
            o = 8 * torch.rand(B, D, device=dev, generator=g) - 4
            obj = FusedObjective("rot_rastrigin", sums={"s": "y**2 - 10 * cos(2 * pi * y)"}, value="10 * D + s", transform=(M, o))
            X = (o[:, None, :] + torch.randn(B, popsize(D), D, device=dev, generator=g)).contiguous()
            obj.evaluate_batched(X)
            torch.cuda.synchronize()
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(5):
                obj.evaluate_batched(X)
            stop.record()
            stop.synchronize()
            calls = max(5, int(50.0 / max(start.elapsed_time(stop) / 5, 1e-3)))
            times = []
            for _ in range(windows):
                start.record()
                for _ in range(calls):
                    obj.evaluate_batched(X)
                stop.record()
                stop.synchronize()
                times.append(start.elapsed_time(stop) / calls)
            out[f"{B}x{D}"] = statistics.median(times)
    return out


def card() -> dict:
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = (v.strip() for v in q.split(","))
    except Exception as e:  # the number is still reported, without the power limit
        out["power_limit"] = f"unread ({type(e).__name__})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.build:
        from evotorch_b200 import build

        for tag, define in VARIANTS.values():
            print(build.build(defines=(define,), tag=tag))
        return
    if a.worker:
        print(json.dumps(worker(a.worker, a.windows)))
        return
    libdir = os.path.join(ROOT, "evotorch_b200", "lib")
    runs = {k: [] for k in VARIANTS}
    for _ in range(a.rounds):
        for k, (tag, _) in VARIANTS.items():
            r = subprocess.run([sys.executable, __file__, "--worker", os.path.join(libdir, f"libevok_{tag}.so"), "--windows", str(a.windows)],
                               capture_output=True, text=True, check=True)
            runs[k].append(json.loads(r.stdout.strip().splitlines()[-1]))
    keys = list(runs["gemm"][0])
    table = []
    for key in keys:
        B, D = (int(v) for v in key.split("x"))
        g = statistics.median(r[key] for r in runs["gemm"])
        f = statistics.median(r[key] for r in runs["fused"])
        table.append({"B": B, "n": popsize(D), "D": D, "gemm_ms": g, "fused_ms": f, "fused_over_gemm": f / g,
                      "spread_gemm": [min(r[key] for r in runs["gemm"]), max(r[key] for r in runs["gemm"])],
                      "spread_fused": [min(r[key] for r in runs["fused"]), max(r[key] for r in runs["fused"])]})
    res = {"card": card(), "sweep": table}
    for row in table:
        print(f"B={row['B']:5d} n={row['n']:3d} D={row['D']:4d}  gemm {row['gemm_ms']:.4f} ms  fused {row['fused_ms']:.4f} ms  "
              f"fused/gemm {row['fused_over_gemm']:.2f}")
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
