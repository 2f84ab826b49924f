"""Time the gradient pass over a materialised population for every read / rebuild split:
python scripts/grad_hybrid_bench.py [POPSIZE DIM [LAUNCHES]]   (default: the metric size, 1M x 10k, 20 launches)

The population is drawn by the fused sampler (Philox + Rastrigin) and ranked with centered utilities, as in a PGPE
generation.  Each variant is timed with CUDA events over LAUNCHES back-to-back launches after 3 warm-up launches:
`grad` (every + row read from HBM), `grad_regen` (every row rebuilt by the lazy population's LDG kernel, an upper bound on
the cost of rebuilding), and `grad_hybrid` at split 0 .. 16 rebuilt row groups per 16 and at the automatic split.  Every
hybrid result must be torch.equal to split 0.  Prints one JSON line; this is how the automatic split was chosen."""
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from evotorch_b200 import ops  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ("?", "?", "?")
    return {"name": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power, "max_sm_clock": clock,
            "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}


def timed(fn, launches: int) -> float:
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    d = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
    launches = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    dev = torch.device("cuda", 0)
    seed, stream_id, form = 7, 3, ops.GRAD_SYMMETRIC
    gen = torch.Generator(device=dev).manual_seed(0)
    mu = (torch.rand(d, device=dev, generator=gen) * 10.24 - 5.12).contiguous()
    sigma = torch.full((d,), 1.0, device=dev)
    X = torch.empty(n, d, device=dev)
    f = torch.empty(n, device=dev)
    ops.sample_eval(ops.OBJ_RASTRIGIN, X, mu, sigma, n_rows=n, symmetric=True, seed=seed, stream_id=stream_id, f=f)
    w = ops.rank(f, "centered", False)
    scale = 2.0 / n
    kw = dict(seed=seed, stream_id=stream_id, row0=0, scale_mu=scale, scale_sigma=scale)

    ref = ops.grad(form, X, w, mu, sigma, scale, scale)
    out = {"popsize": n, "dim": d, "launches": launches, "card": card(), "ms": {}, "equal_to_split0": {}}
    out["ms"]["grad"] = timed(lambda: ops.grad(form, X, w, mu, sigma, scale, scale), launches)
    out["ms"]["grad_regen"] = timed(lambda: ops.grad_regen(form, w, mu, sigma, **kw), launches)
    base = ops.grad_hybrid(form, X, w, mu, sigma, split=0, **kw)
    out["split0_equal_to_grad"] = bool(torch.equal(base[0], ref[0]) and torch.equal(base[1], ref[1]))
    for split in list(range(ops.GRAD_SPLIT_PERIOD + 1)) + [-1]:
        key = "auto" if split < 0 else str(split)
        out["ms"][f"grad_hybrid_{key}"] = timed(lambda: ops.grad_hybrid(form, X, w, mu, sigma, split=split, **kw), launches)
        g = ops.grad_hybrid(form, X, w, mu, sigma, split=split, **kw)
        out["equal_to_split0"][key] = bool(torch.equal(g[0], base[0]) and torch.equal(g[1], base[1]))
    out["ms"] = {k: round(v, 4) for k, v in out["ms"].items()}
    out["all_equal"] = out["split0_equal_to_grad"] and all(out["equal_to_split0"].values())
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
