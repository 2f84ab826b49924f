"""Summarise .ncu-rep captures (read here, no GPU needed) into small CSV files next to them.

    python scripts/ncu_summary.py <tag> [capture directory, default ncu_captures/ (git-ignored)]
"""
import csv
import io
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG = sys.argv[1] if len(sys.argv) > 1 else "r01"
KEEP = ("gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
        "launch__waves_per_multiprocessor", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__cycles_elapsed.avg.per_second", "lts__t_sector_hit_rate.pct", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "smsp__inst_executed_op_shared_ld.sum")


def summarise(rep, out, title):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    if len(rows) < 3:
        print("no data in", rep)
        return
    hdr, units, vals = rows[0], rows[1], rows[-1]
    with open(out, "w") as f:
        f.write(f"# {title}\n# source: {os.path.basename(rep)} (ncu --set full --clock-control none --import-source on)\n")
        f.write(f"# kernel: {vals[hdr.index('Kernel Name')]}\n")
        for i, h in enumerate(hdr):
            if h in KEEP or ("issue_stalled" in h and "per_issue_active" in h) or (("pipe_tensor" in h or "pipe_tmem" in h) and ".avg" in h):
                f.write(f"{h},{units[i]},{vals[i]}\n")
    print("wrote", out)


def launch_shares(csv_path, out):
    rows = list(csv.reader(open(csv_path)))
    start = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    h = rows[start]
    ki, vi = h.index("Kernel Name"), h.index("Metric Value")
    agg = defaultdict(lambda: [0, 0.0])
    for r in rows[start + 1:]:
        if len(r) <= vi:
            continue
        try:
            v = float(r[vi].replace(",", ""))
        except ValueError:
            continue
        name = r[ki].split("(")[0][:90]
        agg[name][0] += 1
        agg[name][1] += v
    tot = sum(v[1] for v in agg.values())
    with open(out, "w") as f:
        f.write("# per-kernel device time of `python bench.py --steps 3 --warmup 3 --no-e2e --no-cpu-baseline` under\n")
        f.write("# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised: compare SHARES)\n")
        f.write("kernel,launches,total_us,share_pct\n")
        for n, (c, t) in sorted(agg.items(), key=lambda x: -x[1][1]):
            f.write(f"\"{n}\",{c},{t / 1e3:.1f},{100 * t / tot:.2f}\n")
    print("wrote", out)


G = P = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "ncu_captures")
os.makedirs(P, exist_ok=True)
for rep, name, title in (("prof_sample_eval", "ncu_sample_eval", "fused Philox sample + Rastrigin evaluate kernel (PGPE 1M x 10k (metric size))"),
                         ("prof_grad", "ncu_grad", "TMA-staged weighted column reduction kernel (PGPE 1M x 10k (metric size))"),
                         ("prof_scatter", "ncu_radix_scatter", "radix sort scatter pass (N = 1M keys)"),
                         ("prof_mlp", "ncu_mlp_forward", "batched MLP policy forward (65536 x 100881)"),
                         ("prof_gemm", "ncu_gemm_tf32x3", "wgmma 3xTF32 GEMM, 4096 x 1024 x 1024 (CMA-ES Y = Z A^T)")):
    path = os.path.join(G, rep + ".ncu-rep")
    if os.path.exists(path):
        summarise(path, os.path.join(P, f"{TAG}_{name}.csv"), title)
if os.path.exists(os.path.join(G, "launches.csv")):
    launch_shares(os.path.join(G, "launches.csv"), os.path.join(P, f"{TAG}_launch_shares.csv"))
