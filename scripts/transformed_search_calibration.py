"""The thresholds of the search-level check of transformed objectives (tests/test_transformed_objective_gpu.py,
test_rotation_reaches_the_search), derived in float64 on the CPU through the torch path.

    python scripts/transformed_search_calibration.py [--items 64] [--out results/transformed_search_calibration.json]

Rotated ellipsoid of condition 1e6, D = 10, a per-item rotation R_b (QR of a Gaussian matrix) and offset o_b in [-4, 4)^10, and its
unrotated twin (the identity transform, same o_b).  Full and separable CMA-ES from the origin with stdev 3 and the default popsize;
the share of items whose best f so far (fmin: a converged search's later NaN rows do not erase it) is below 1e-4 and 1e-6 after
the listed generations.  The GPU test uses G = 600 and tau = 1e-4 (f at the optimum resolves to about 2.5e-7 per float32 ulp of x)
and asks for a share of at least 0.9 where the family fits, at most 0.1 where it does not.
"""

import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask_and_evaluate, cmaes_tell, sepcmaes,  # noqa: E402
                                                 sepcmaes_ask_and_evaluate, sepcmaes_tell)
from evotorch_b200.objectives import FusedObjective  # noqa: E402

CHECKPOINTS = (200, 300, 400, 500, 600, 800, 1000, 1200)
TAUS = (1e-4, 1e-6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.manual_seed(0)
    B, D = a.items, 10
    R = torch.linalg.qr(torch.randn(B, D, D, dtype=torch.float64))[0].float()
    o = 8 * torch.rand(B, D) - 4
    eye = torch.eye(D).expand(B, D, D).contiguous()
    res = {}
    for name, M in (("rotated", R), ("unrotated", eye)):
        obj = FusedObjective("ell", sums={"s": "10**(6 * j / (D - 1)) * y**2"}, value="s", transform=(M, o))
        for fam, (make, ask, tell) in (("full", (cmaes, cmaes_ask_and_evaluate, cmaes_tell)),
                                       ("separable", (sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell))):
            state = make(center_init=torch.zeros(B, D, dtype=torch.float64), stdev_init=3.0, objective_sense="min")
            best = torch.full((B,), math.inf, dtype=torch.float64)
            shares = {}
            for g in range(1, CHECKPOINTS[-1] + 1):
                values, evals = ask(state, objective=obj)
                state = tell(state, values, evals)
                best = torch.fmin(best, evals.min(-1).values)
                if g in CHECKPOINTS:
                    shares[g] = {str(t): (best < t).double().mean().item() for t in TAUS}
            res[f"{fam}_{name}"] = shares
            print(fam, name, json.dumps(shares), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"items": B, "dtype": "float64", "device": "cpu", "shares": res}, fh, indent=1)


if __name__ == "__main__":
    main()
