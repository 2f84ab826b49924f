"""Float64 restatement of the functional ask / tell API's tells  --  TEST INFRASTRUCTURE ONLY.

One batch item at a time, what `pgpe_tell`, `cem_tell` and the `clipup_tell` / `adam_tell` / `sgd_tell` of
`evotorch_b200.algorithms.functional` compute (reference: algorithms/functional/funcpgpe.py, funccem.py, funcclipup.py,
funcadam.py, funcsgd.py).  Built from the pieces of `es_oracle` that the reference pins (tests/test_oracle_golden.py): the
rankings and their stable order, the ClipUp / Adam update rules and `modify_tensor` with its NaN propagation; only the weighted
sums, the elite moments and the functional momentum step are new here, and those are evaluated in float64.

Besides each result, the gradient functions return its MAGNITUDE: the same sum evaluated on absolute values, which is what a
float32 evaluation's rounding error is proportional to (tests bound |x32 - x64| by c * 2^-24 * K_eff * magnitude).
Checked against the real reference's outputs (tests/golden/functional_golden.npz) and against the package's own torch path run in
float64 on the CPU: tests/test_functional_oracle.py.
"""

from __future__ import annotations

import math
from typing import Optional

import numpy as np

from . import es_oracle as O

F64 = np.float64


def _f64(x) -> np.ndarray:
    return np.asarray(x, dtype=F64)


# ------------------------------------------------------------------------------------------------ ranking
def utilities(evals, ranking_method: str, maximize: bool) -> np.ndarray:
    """The utilities pgpe_tell weights the population with: `es_oracle.rank` (fp32, as the reference and the kernels produce
    them), then w - mean(w) in float64 for the rankings that are not already centred (distributions.py:562-563, :722-723)."""
    w = O.rank(np.asarray(evals, dtype=np.float32), ranking_method, maximize).astype(F64)
    if ranking_method not in ("centered", "normalized"):
        w = w - w.mean()
    return w


def elite_indices(evals, num_elites: int, maximize: bool) -> np.ndarray:
    """The `num_elites` best solutions, best first; ties in ascending index (the stable order of `argsort_for_ranking`)."""
    w = O.rank_raw(evals, maximize)
    return O.argsort_for_ranking(w, higher_is_better=False)[: int(num_elites)]


# ------------------------------------------------------------------------------------------------ weighted sums
GRAD_SEPARABLE, GRAD_SYMMETRIC, GRAD_EXP, GRAD_MOMENTS = 0, 1, 2, 3  # the forms of include/evok.h


def weighted_sums(form: int, values, w, center, stdev, w_mag=None) -> dict:
    """S1_j = sum_r a_r eps_rj and S2_j = sum_r b_r g(eps_rj) of one item, eps = x - mu, for the four gradient forms of
    include/evok.h: SEPARABLE g = (eps^2 - sigma^2) / sigma, a = b = w; SYMMETRIC the same g over the even rows with
    a, b = (w+ -+ w-) / 2; EXP g = (eps / sigma)^2 - 1; MOMENTS g = eps^2.  `w_mag` (default |w|) bounds the error of the weights
    themselves.  Returns {"s1", "s2", "s1_mag", "s2_mag"}."""
    X, mu, sigma, w = _f64(values), _f64(center), _f64(stdev), _f64(w)
    wm = np.abs(w) if w_mag is None else _f64(w_mag)
    if form == GRAD_SYMMETRIC:
        eps = X[0::2] - mu
        a, b = (w[0::2] - w[1::2]) / 2, (w[0::2] + w[1::2]) / 2
        am = bm = (wm[0::2] + wm[1::2]) / 2
    else:
        eps = X - mu
        a = b = w
        am = bm = wm
    if form in (GRAD_SEPARABLE, GRAD_SYMMETRIC):
        g, gm = (eps * eps - sigma * sigma) / sigma, (eps * eps + sigma * sigma) / np.abs(sigma)
    elif form == GRAD_EXP:
        g, gm = (eps / sigma) ** 2 - 1, (eps / sigma) ** 2 + 1
    else:
        g = gm = eps * eps
    return {"s1": a @ eps, "s2": b @ g, "s1_mag": am @ np.abs(eps), "s2_mag": bm @ gm}


# ------------------------------------------------------------------------------------------------ PGPE
def pgpe_gradients(values, evals, center, stdev, *, ranking_method: str, maximize: bool, symmetric: bool) -> dict:
    """grad_mu and grad_sigma of one PGPE tell, divided by the number of directions (symmetric) or of solutions (non-symmetric), as
    `pgpe` configures its distributions.  Symmetric: rows (2k, 2k+1) are the antithetic pair mu +- eps_k, weighted by
    (w+ - w-) / 2 and (w+ + w-) / 2.  Returns {"mu", "sigma", "mu_mag", "sigma_mag", "w"}; the magnitudes count the fp32 rounding
    of w - mean(w) against the weights before the subtraction."""
    w = utilities(evals, ranking_method, maximize)
    w_mag = np.abs(w)
    if ranking_method not in ("centered", "normalized"):
        raw = O.rank(np.asarray(evals, dtype=np.float32), ranking_method, maximize).astype(F64)
        w_mag = np.abs(w) + np.abs(raw).max()
    n = len(w)
    scale = 1.0 / (n // 2) if symmetric else 1.0 / n
    s = weighted_sums(GRAD_SYMMETRIC if symmetric else GRAD_SEPARABLE, values, w, center, stdev, w_mag)
    return {"mu": scale * s["s1"], "sigma": scale * s["s2"], "mu_mag": scale * s["s1_mag"], "sigma_mag": scale * s["s2_mag"], "w": w}


def sigma_update(stdev, grad_sigma, lr: float, *, exp_form: bool = False, stdev_min=None, stdev_max=None, stdev_max_change=None) -> tuple:
    """(new stdev, target) of the stdev step: target = stdev + lr * grad (`exp_form`: stdev * exp(lr * grad / 2), SNES), then
    `es_oracle.modify_tensor` against the old stdev
    (a NaN target, bound or allowed change |0| * inf gives NaN, as torch.max / torch.min).  The target is rounded to fp32 before the
    clamp: a clamp moves no value by more than the target's own error."""
    step = float(lr) * _f64(grad_sigma)
    target = _f64(stdev) * np.exp(0.5 * step) if exp_form else _f64(stdev) + step
    new = O.modify_tensor(stdev, target.astype(np.float32), lb=stdev_min, ub=stdev_max, max_change=stdev_max_change)
    return new.astype(F64), target


# ------------------------------------------------------------------------------------------------ CEM
def cem_moments(values, evals, center, *, parenthood_ratio: float, maximize: bool) -> dict:
    """Elite mean and unbiased elite std of one CEM tell, two-pass in float64 (E = floor(N * ratio) elites).  As torch.mean /
    torch.std: E = 0 gives NaN for both, E = 1 a NaN std.  Also the kernels' intermediate quantities: S1 = sum (x - mu) and
    S2 = sum (x - mu)^2 over the elites, with their magnitudes."""
    X, mu = _f64(values), _f64(center)
    num_elites = int(math.floor(X.shape[0] * float(parenthood_ratio)))
    idx = elite_indices(evals, num_elites, maximize)
    elites = X[idx]
    nan = np.full(X.shape[1], np.nan)
    mean = elites.mean(axis=0) if num_elites >= 1 else nan
    std = np.sqrt(((elites - mean) ** 2).sum(axis=0) / (num_elites - 1)) if num_elites >= 2 else nan
    eps = elites - mu
    return {"mean": mean, "std": std, "num_elites": num_elites, "elite_indices": idx, "s1": eps.sum(axis=0), "s2": (eps * eps).sum(axis=0),
            "s1_mag": np.abs(eps).sum(axis=0)}


def cem_tell(values, evals, center, stdev, *, parenthood_ratio: float, maximize: bool, stdev_min=None, stdev_max=None,
             stdev_max_change=None) -> dict:
    """center <- mean(elites); stdev <- modify_tensor(stdev, std(elites), ...).  Returns the moments plus "center" and "stdev"."""
    mom = cem_moments(values, evals, center, parenthood_ratio=parenthood_ratio, maximize=maximize)
    new_stdev, _ = sigma_update(stdev, mom["std"] - _f64(stdev), 1.0, stdev_min=stdev_min, stdev_max=stdev_max,
                                stdev_max_change=stdev_max_change)
    return dict(mom, center=mom["mean"], stdev=new_stdev)


# ------------------------------------------------------------------------------------------------ functional optimizers
def clipup_tell(center, velocity, grad, *, lr: float, momentum: float, max_speed: float) -> dict:
    """`es_oracle.ClipUp` from the given velocity: v <- clip(momentum v + lr g / ||g||, max_speed); center <- center + v.
    Also returns the unclipped speed, so that tests can keep clear of the clip threshold."""
    opt = O.ClipUp(len(center), lr, momentum, max_speed)
    opt.velocity = np.asarray(velocity, dtype=np.float32).copy()
    g = np.asarray(grad, dtype=np.float32)
    g64 = g.astype(F64)
    unclipped = momentum * _f64(velocity) + lr * g64 / np.linalg.norm(g64)
    v = opt.ascent(g).astype(F64)
    return {"center": _f64(center) + v, "velocity": v, "speed": float(np.linalg.norm(unclipped)),
            "clipped": bool(np.linalg.norm(unclipped) > max_speed)}


def adam_tell(center, m, v, t: int, grad, *, lr: float, beta1: float = 0.9, beta2: float = 0.999, epsilon: float = 1e-8) -> dict:
    """`es_oracle.Adam` from the given moments and step count t (t + 1 after this tell)."""
    opt = O.Adam(len(center), lr, beta1, beta2, epsilon)
    opt.m, opt.v, opt.t = np.asarray(m, np.float32).copy(), np.asarray(v, np.float32).copy(), int(t)
    step = opt.ascent(grad).astype(F64)
    return {"center": _f64(center) + step, "m": opt.m.astype(F64), "v": opt.v.astype(F64), "t": opt.t, "step": step}


def sgd_tell(center, velocity, grad, *, lr: float, momentum: Optional[float] = None) -> dict:
    """velocity <- momentum velocity + lr g; center <- center + velocity.  With a constant lr this is `es_oracle.SGD` (buffer
    b <- momentum b + g, step lr b) with velocity = lr b, written in the functional API's own state."""
    mom = 0.0 if momentum is None else float(momentum)
    vel = mom * _f64(velocity) + float(lr) * _f64(grad)
    return {"center": _f64(center) + vel, "velocity": vel}
