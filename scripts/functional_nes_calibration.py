"""The budget of the search-level check of XNES and SNES (tests/test_functional_nes_gpu.py, test_search_outcome), derived in
float64 on the CPU through the torch path.

    python scripts/functional_nes_calibration.py [--items 32] [--out results/functional_nes_calibration.json]

D = 16, a per-item rotation R_b (QR of a Gaussian matrix) and offset o_b in [-4, 4)^16, the rotated ellipsoid
sum_j 10^(4 j / (D - 1)) y_j^2 of y = R_b (x - o_b) (condition 1e4).  XNES, which learns the rotation, and SNES, which cannot,
from the origin with stdev 2 and their default popsizes; the share of items whose best f so far is below 1e-6 after the listed
generations.
"""

import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evotorch_b200.algorithms.functional import snes, snes_ask_and_evaluate, snes_tell, xnes, xnes_ask_and_evaluate, xnes_tell  # noqa: E402
from evotorch_b200.objectives import FusedObjective  # noqa: E402

D = 16
TAU = 1e-6
CHECKPOINTS = (500, 1000, 1500, 2000, 2500, 3000, 4000, 5000)
FAMILIES = {"xnes": (xnes, xnes_ask_and_evaluate, xnes_tell), "snes": (snes, snes_ask_and_evaluate, snes_tell)}


def problem(B: int, dtype=torch.float32, device="cpu") -> FusedObjective:
    """The rotated ellipsoid with the per-item rotations and offsets of seed 0."""
    g = torch.Generator().manual_seed(0)
    R = torch.linalg.qr(torch.randn(B, D, D, generator=g, dtype=torch.float64))[0].to(dtype=dtype, device=device)
    o = (8 * torch.rand(B, D, generator=g, dtype=torch.float64) - 4).to(dtype=dtype, device=device)
    return FusedObjective("nes_ellipsoid", sums={"s": "10**(4 * j / (D - 1)) * y**2"}, value="s", transform=(R, o))


def shares(family: str, obj, B: int, checkpoints, dtype=torch.float64, device="cpu") -> dict:
    make, ask, tell = FAMILIES[family]
    state = make(center_init=torch.zeros(B, D, dtype=dtype, device=device), stdev_init=2.0, objective_sense="min")
    best = torch.full((B,), math.inf, dtype=dtype, device=device)
    out = {}
    for g in range(1, checkpoints[-1] + 1):
        values, evals = ask(state, objective=obj)
        state = tell(state, values, evals)
        best = torch.fmin(best, evals.min(-1).values)
        if g in checkpoints:
            out[g] = (best < TAU).double().mean().item()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.manual_seed(0)
    obj = problem(a.items)
    res = {}
    for fam in FAMILIES:
        res[fam] = shares(fam, obj, a.items, CHECKPOINTS)
        print(fam, json.dumps(res[fam]), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"items": a.items, "D": D, "tau": TAU, "condition": 1e4, "dtype": "float64", "device": "cpu", "shares": res}, fh, indent=1)


if __name__ == "__main__":
    main()
