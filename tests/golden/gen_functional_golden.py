"""Golden vectors for the functional (ask/tell) API, produced by running the REAL reference
(`evotorch.algorithms.functional`, reference files funcpgpe.py / funccem.py / funcclipup.py / funcadam.py / funcsgd.py):

    PYTHONPATH=tests/golden/_refstubs:/root/reference/src EVOTORCH_VERBOSE_LEVEL=0 python tests/golden/gen_functional_golden.py

CPU, float32.  The populations the reference drew (`*_ask`, torch's global RNG) are stored next to the states that
`*_tell` produced from them, so the tests replay the tells on identical inputs.
"""

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

import evotorch  # noqa: E402  (the reference)
from evotorch.algorithms.functional import (  # noqa: E402
    adam, adam_ask, adam_tell, cem, cem_ask, cem_tell, clipup, clipup_ask, clipup_tell, pgpe, pgpe_ask, pgpe_tell, sgd, sgd_ask, sgd_tell,
)

assert "/root/reference" in evotorch.__file__, evotorch.__file__
torch.manual_seed(20240921)
rng = np.random.default_rng(77)
out = {}


def T(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.float32)


def npy(t):
    return t.detach().cpu().numpy().copy()


def rastrigin(x):
    return 10 * x.shape[-1] + torch.sum(x**2 - 10 * torch.cos(2 * np.pi * x), dim=-1)


# ---------------------------------------------------------------- functional optimizers
D = 7
grads = rng.standard_normal((5, D)).astype(np.float32)
grads_b = rng.standard_normal((5, 3, D)).astype(np.float32)
c0 = rng.standard_normal(D).astype(np.float32)
c0_b = rng.standard_normal((3, D)).astype(np.float32)
out["opt/grads"], out["opt/grads_b"], out["opt/c0"], out["opt/c0_b"] = grads, grads_b, c0, c0_b

cases = {
    "clipup": (clipup, clipup_ask, clipup_tell, dict(center_learning_rate=0.15, momentum=0.9), dict(center_learning_rate=T([0.1, 0.2, 0.3]), max_speed=T([0.15, 0.5, 0.45]))),
    "adam": (adam, adam_ask, adam_tell, dict(center_learning_rate=0.05), dict(center_learning_rate=T([0.01, 0.05, 0.1]), beta1=0.8)),
    "sgd": (sgd, sgd_ask, sgd_tell, dict(center_learning_rate=0.1, momentum=0.5), dict(center_learning_rate=T([0.1, 0.2, 0.3]))),
}
for name, (init, ask, tell, cfg, cfg_b) in cases.items():
    for tag, start, gs, kw in (("plain", c0, grads, cfg), ("batched", c0_b, grads_b, cfg_b)):
        st = init(center_init=T(start), **kw)
        centers = []
        for g in gs:
            st = tell(st, follow_grad=T(g))
            centers.append(npy(ask(st)))
        out[f"opt/{name}/{tag}/centers"] = np.stack(centers)

# ---------------------------------------------------------------- functional PGPE
D, N, G = 12, 40, 4
pg_cases = {
    "sym_clipup": dict(kw=dict(center_learning_rate=0.3, stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0), batch=()),
    "nonsym_adam_nes": dict(kw=dict(center_learning_rate=0.05, stdev_learning_rate=0.1, objective_sense="min", stdev_init=0.7, optimizer="adam",
                                    ranking_method="nes", symmetric=False, stdev_max_change=None), batch=()),
    "sym_sgd_linear_max": dict(kw=dict(center_learning_rate=0.1, stdev_learning_rate=0.2, objective_sense="max", radius_init=3.0, optimizer="sgd",
                                       ranking_method="linear", stdev_min=0.5, stdev_max=1.0, stdev_max_change=0.1), batch=()),
    "batched": dict(kw=dict(center_learning_rate=T([0.2, 0.4]), stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0), batch=(2,)),
}
for tag, case in pg_cases.items():
    center0 = T(rng.uniform(-3, 3, size=case["batch"] + (D,)))
    st = pgpe(center_init=center0, **case["kw"])
    out[f"pgpe/{tag}/center0"], out[f"pgpe/{tag}/stdev0"] = npy(center0), npy(st.stdev)
    rec = {"values": [], "evals": [], "center": [], "stdev": []}
    for _ in range(G):
        values = pgpe_ask(st, popsize=N)
        evals = rastrigin(values)
        st = pgpe_tell(st, values, evals)
        rec["values"].append(npy(values)); rec["evals"].append(npy(evals))
        rec["center"].append(npy(st.optimizer_state.center)); rec["stdev"].append(npy(st.stdev))
    for k, v in rec.items():
        out[f"pgpe/{tag}/{k}"] = np.stack(v)

# ---------------------------------------------------------------- functional CEM
cem_cases = {
    "plain": dict(kw=dict(parenthood_ratio=0.25, objective_sense="min", stdev_init=2.0, stdev_max_change=0.3), batch=()),
    "max_bounds": dict(kw=dict(parenthood_ratio=0.5, objective_sense="max", stdev_init=1.0, stdev_min=0.4, stdev_max=1.5), batch=()),
    "batched": dict(kw=dict(parenthood_ratio=0.25, objective_sense="min", stdev_init=T([[1.0] * D, [2.0] * D, [0.5] * D])), batch=(3,)),
}
for tag, case in cem_cases.items():
    center0 = T(rng.uniform(-3, 3, size=case["batch"] + (D,)))
    st = cem(center_init=center0, **case["kw"])
    out[f"cem/{tag}/center0"], out[f"cem/{tag}/stdev0"] = npy(center0), npy(st.stdev)
    rec = {"values": [], "evals": [], "center": [], "stdev": []}
    for _ in range(G):
        values = cem_ask(st, popsize=N)
        evals = rastrigin(values)
        st = cem_tell(st, values, evals)
        rec["values"].append(npy(values)); rec["evals"].append(npy(evals)); rec["center"].append(npy(st.center)); rec["stdev"].append(npy(st.stdev))
    for k, v in rec.items():
        out[f"cem/{tag}/{k}"] = np.stack(v)

# ---------------------------------------------------------------- functional CEM at its edges (one tell each; drawn after every case
# above, so the keys above do not change).  One elite: std of one row is NaN.  No elite: mean and std of no rows are NaN.  A zero in
# `stdev_init` with the default stdev_max_change=None (inf): the allowed change |0| * inf is NaN, and torch.max / torch.min keep it.
cem_edge_cases = {
    "one_elite": dict(kw=dict(parenthood_ratio=0.03, objective_sense="min", stdev_init=1.0), batch=()),
    "zero_elites": dict(kw=dict(parenthood_ratio=0.01, objective_sense="max", stdev_init=1.0), batch=()),
    "zero_stdev": dict(kw=dict(parenthood_ratio=0.25, objective_sense="min", stdev_init=T([1.0, 0.0] * (D // 2))), batch=()),
}
for tag, case in cem_edge_cases.items():
    center0 = T(rng.uniform(-3, 3, size=case["batch"] + (D,)))
    st = cem(center_init=center0, **case["kw"])
    out[f"cem/{tag}/center0"], out[f"cem/{tag}/stdev0"] = npy(center0), npy(st.stdev)
    values = cem_ask(st, popsize=N)
    evals = rastrigin(values)
    st = cem_tell(st, values, evals)
    for k, v in (("values", values), ("evals", evals), ("center", st.center), ("stdev", st.stdev)):
        out[f"cem/{tag}/{k}"] = npy(v)[None]

np.savez_compressed(os.path.join(HERE, "functional_golden.npz"), **out)
print("wrote", len(out), "arrays ->", os.path.join(HERE, "functional_golden.npz"), file=sys.stderr)
