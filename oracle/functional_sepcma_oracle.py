"""Float64 reference for the batched functional separable CMA-ES (`algorithms/functional/funcsepcmaes.py`), shared by its tests.

* `item_state`: one item of a state as a `SepItem` (float64 arrays of its values, the learning rates and weights of the state).
* `reference_generation`: one separable generation of one item (cmaes.py:432-565 of the reference with separable=True, and
  `_limit_stdev`, cmaes.py:49-79), fed the item's own values and fitnesses: the steps are recovered from the values,
  z = (x - m) / s, as the functional tell recovers them.  Optionally with one of `MUTATIONS`: the wrong algorithms a batched
  implementation can plausibly compute, which the tests must tell apart from the right one.
* `generation_bound`: the first-order bound of a tell computed with unit roundoff `eps` against that reference, per output.
* `tell_ratios`: per item, the largest |tell - reference| / (2 bound) over the new state.
"""

from __future__ import annotations

import copy
import math

import numpy as np
import torch

EPS32 = 2.0 ** -24
EPS64 = 2.0 ** -53

# "neighbour_fitness": item b is ranked with item b+1's fitnesses (applied by `tell_ratios`, which owns the batch); "raw_z": the
# moments over the drawn z instead of the steps recovered from the (repaired) values; "q_other_z": the active weights divide by
# the squared norm of the drawn z, not of the recovered one; "no_active": active weights off; "wsum_positive": wsum = the sum of
# the positive weights; "clamp_old_sigma": the stdev bounds with the sigma from before the generation; "decompose_off_by_one":
# A <- sqrt(C) when steps % freq == 0 instead of (steps + 1) % freq == 0
MUTATIONS = ("neighbour_fitness", "raw_z", "q_other_z", "no_active", "wsum_positive", "clamp_old_sigma", "decompose_off_by_one")

FIELDS = ("m", "sigma", "C", "A", "s", "p_sigma", "p_c")


class SepItem:
    """One separable search: its state (float64 arrays) and the hyper-parameters of the state it came from."""

    def __init__(self, hp, d: int, *, active: bool, csa_squared: bool, stdev_min, stdev_max):
        self.d, self.popsize = int(d), hp.popsize
        self.weights = hp.weights.detach().cpu().numpy().astype(np.float64)
        self.c_m, self.c_sigma, self.damp_sigma, self.c_c, self.c_1, self.c_mu = hp.c_m, hp.c_sigma, hp.damp_sigma, hp.c_c, hp.c_1, hp.c_mu
        self.vd_sigma, self.vd_c, self.unbiased_expectation = hp.variance_discount_sigma, hp.variance_discount_c, float(hp.unbiased_expectation)
        self.decompose_C_freq = hp.decompose_C_freq
        self.active, self.csa_squared, self.stdev_min, self.stdev_max = active, csa_squared, stdev_min, stdev_max


def stable_ranks(f, descending: bool) -> np.ndarray:
    """Position of each key in the stable order (position 0 = the largest key if `descending`), in the keys' own precision: ties
    keep ascending index order in both senses, -0 and +0 are equal, NaN is larger than +inf (the order of rank_table and of the
    torch tell's stable argsort)."""
    f = np.asarray(f)
    nan = np.isnan(f)
    if descending:
        order = np.lexsort((np.where(nan, 0.0, -f.astype(np.float64)), ~nan))  # sorts by its last key first: NaN first
    else:
        order = np.argsort(f, kind="stable")
    ranks = np.empty(len(f), dtype=np.int64)
    ranks[order] = np.arange(len(f))
    return ranks


def item_state(state, b: int) -> SepItem:
    """Item b (flat index over the batch dimensions) of a SepCMAESState."""
    d = state.center.shape[-1]
    o = SepItem(state.hyperparameters, d, active=state.active, csa_squared=state.csa_squared, stdev_min=state.stdev_min, stdev_max=state.stdev_max)
    for name, t in (("m", state.center), ("C", state.C), ("A", state.A), ("s", state.s), ("p_sigma", state.p_sigma), ("p_c", state.p_c)):
        setattr(o, name, t.detach().reshape(-1, d)[b].cpu().double().numpy().copy())
    o.sigma = float(state.sigma.reshape(-1)[b])
    o.steps = state.generation
    return o


def reference_generation(o: SepItem, X, f, sense: str, mutation=None, z_raw=None) -> dict:
    """One generation of item `o` (updated in place) from its values X (n, D) and fitnesses f (n,).  Returns the intermediate
    quantities the bound needs: the steps z, the weights a, b and their aw, the moments, h_sig and the margin of its comparison."""
    X = np.asarray(X, np.float64)
    d = o.d
    z = (X - o.m) / o.s
    if mutation in ("raw_z", "q_other_z") and z_raw is None:
        raise ValueError(f"the mutation {mutation!r} needs the drawn z")
    zs = np.asarray(z_raw, np.float64) if mutation == "raw_z" else z
    zq = np.asarray(z_raw, np.float64) if mutation == "q_other_z" else z
    aw = o.weights[stable_ranks(f, sense == "max")]
    a = np.maximum(aw, 0.0)
    q = (zq * zq).sum(axis=1)
    active = o.active and mutation != "no_active"
    with np.errstate(divide="ignore", invalid="ignore"):
        b = np.where(aw < 0, d * aw / q, aw) if active else aw.copy()
    local, S2 = a @ zs, b @ (zs * zs)
    wsum = float(a.sum()) if mutation == "wsum_positive" else float(b.sum())
    # the update (cmaes.py:454-565, separable branch): shaped = A * local, sum_i b_i y_i^2 = A^2 S2
    sig0 = o.sigma
    shaped = o.A * local
    o.m = o.m + o.c_m * sig0 * shaped
    o.p_sigma = (1 - o.c_sigma) * o.p_sigma + o.vd_sigma * local
    pnorm = float(np.sqrt(np.sum(o.p_sigma**2)))
    expo = (pnorm**2 / d - 1) / 2 if o.csa_squared else pnorm / o.unbiased_expectation - 1
    o.sigma = sig0 * math.exp((o.c_sigma / o.damp_sigma) * expo)
    squared_sum = pnorm**2 / (1 - (1 - o.c_sigma) ** (2 * o.steps + 1))
    margin = (1 + 4.0 / (d + 1)) - ((squared_sum / d) - 1)
    h = 1.0 if margin > 0 else 0.0
    p_c_old = o.p_c
    o.p_c = (1 - o.c_c) * o.p_c + h * o.vd_c * shaped
    c1a = o.c_1 * (1 - (1 - h**2) * o.c_c * (2 - o.c_c))
    C_old = o.C
    o.C = o.C + c1a * (o.p_c**2 - o.C) + o.c_mu * (o.A**2 * S2 - wsum * o.C)
    C_unclamped = o.C
    if o.stdev_min is not None or o.stdev_max is not None:
        sg = sig0 if mutation == "clamp_old_sigma" else o.sigma
        stdevs = np.clip(sg * np.sqrt(o.C), o.stdev_min, o.stdev_max)
        o.C = (stdevs / sg) ** 2
    decompose = ((o.steps if mutation == "decompose_off_by_one" else o.steps + 1) % o.decompose_C_freq) == 0
    A_old = o.A
    if decompose:
        o.A = np.sqrt(o.C)
    o.s = o.sigma * o.A
    o.steps += 1
    return dict(z=z, zs=zs, aw=aw, a=a, b=b, q=q, local=local, S2=S2, wsum=wsum, shaped=shaped, h=h, margin=margin, sig0=sig0, pnorm=pnorm,
                p_c_old=p_c_old, C_old=C_old, C_unclamped=C_unclamped, A_old=A_old, decompose=decompose, c1a=c1a)


def generation_bound(before: SepItem, out: dict, after: SepItem, eps: float) -> dict:
    """First-order bound, per output of `FIELDS`, of |tell - reference| for a tell computed in a precision with unit roundoff
    `eps` from the same state, values and fitnesses: z = (x - m) / s with two roundings, the sums of q and of the moments in any
    order (gamma_k = k eps / (1 - k eps)), then the update's few roundings per element, carried through the clamp and the square
    root.  h_sig is taken as exact (the tests check its margin)."""
    u = eps
    d = before.d
    z, a, b, q = out["z"], out["a"], out["b"], out["q"]
    n = z.shape[0]
    gam = lambda k: k * u / (1 - k * u)  # noqa: E731
    az = np.abs(z)
    dz = 3 * u * az
    with np.errstate(divide="ignore", invalid="ignore"):
        dq = gam(d) * q + 2 * (az * dz).sum(axis=1)
        db = np.where(out["aw"] < 0, np.abs(b) * (dq / q + 2 * u), 0.0) if before.active else np.zeros_like(b)
    zz = z * z
    e_loc = gam(n) * (a @ az) + a @ dz
    e_S2 = (gam(n) + 2 * u) * (np.abs(b) @ zz) + db @ zz + np.abs(b) @ (2 * az * dz)
    e_ws = gam(n) * float(np.abs(b).sum()) + float(db.sum())
    A, sig0 = before.A, before.sigma
    e_sh = np.abs(A) * e_loc + u * np.abs(out["shaped"])
    e_m = before.c_m * sig0 * e_sh + 4 * u * (np.abs(before.m) + before.c_m * sig0 * np.abs(out["shaped"]))
    e_ps = before.vd_sigma * e_loc + 4 * u * (np.abs((1 - before.c_sigma) * before.p_sigma) + np.abs(before.vd_sigma * out["local"]))
    e_pn = float(np.sqrt((e_ps**2).sum())) + u * out["pnorm"]
    slope = out["pnorm"] / d if before.csa_squared else 1.0 / before.unbiased_expectation
    sig = after.sigma
    e_sig = sig * ((before.c_sigma / before.damp_sigma) * slope * e_pn + 8 * u)
    e_pc = out["h"] * before.vd_c * e_sh + 4 * u * (np.abs((1 - before.c_c) * out["p_c_old"]) + np.abs(after.p_c))
    C0, c1a = out["C_old"], out["c1a"]
    e_C = (2 * c1a * np.abs(after.p_c) * e_pc + before.c_mu * (A**2 * e_S2 + e_ws * np.abs(C0))
           + 8 * u * (np.abs(C0) + c1a * (after.p_c**2 + np.abs(C0)) + before.c_mu * (A**2 * np.abs(out["S2"]) + abs(out["wsum"]) * np.abs(C0))
                      + np.abs(out["C_unclamped"])))
    if before.stdev_min is not None or before.stdev_max is not None:
        e_C = e_C + np.abs(after.C) * (2 * e_sig / sig + 8 * u)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_A = e_C / (2 * np.sqrt(after.C)) + u * np.abs(after.A) if out["decompose"] else np.zeros(d)
    e_s = np.abs(after.A) * e_sig + sig * e_A + u * np.abs(after.s)
    return dict(m=e_m, sigma=np.asarray(e_sig), C=e_C, A=e_A, s=e_s, p_sigma=e_ps, p_c=e_pc)


def _as_np(t) -> np.ndarray:
    return t.detach().cpu().double().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float64)


def tell_ratios(state, x, f, new, mutation=None, z_raw=None, items=None, record=None) -> list:
    """Per item of `items` (default: all) of `state`: max over the fields of `new` (the told state) of |new - reference| / (2 bound),
    with the reference and bound of one generation from `state`, the values x (..., n, D) and fitnesses f (..., n), in the
    precision of the state's dtype.  z_raw (..., n, D): the drawn z, for the mutations that use it.  `record` (a list) receives each
    item's reference outcome."""
    d, n = state.center.shape[-1], state.popsize
    xs, fs = _as_np(x).reshape(-1, n, d), _as_np(f).reshape(-1, n)
    zr = None if z_raw is None else _as_np(z_raw).reshape(-1, n, d)
    B = xs.shape[0]
    eps = EPS32 if state.center.dtype == torch.float32 else EPS64
    sense = "max" if state.maximize else "min"
    got = {"m": new.center, "sigma": new.sigma, "C": new.C, "A": new.A, "s": new.s, "p_sigma": new.p_sigma, "p_c": new.p_c}
    got = {k: _as_np(v).reshape(B, -1) for k, v in got.items()}
    ratios = []
    for b in (range(B) if items is None else items):
        o = item_state(state, b)
        before = copy.deepcopy(o)
        fb = fs[(b + 1) % B] if mutation == "neighbour_fitness" and B > 1 else fs[b]
        out = reference_generation(o, xs[b], fb, sense, mutation, None if zr is None else zr[b])
        if record is not None:
            record.append(out)
        bound = generation_bound(before, out, o, eps)
        r = 0.0
        for k in FIELDS:
            ref = np.atleast_1d(np.asarray(o.sigma if k == "sigma" else getattr(o, k), np.float64))
            err = np.abs(got[k][b] - ref)
            q = np.where(np.isfinite(err), err / (2 * np.atleast_1d(bound[k]) + 1e-300), np.inf)
            r = max(r, float(q.max()))
        ratios.append(r)
    return ratios
