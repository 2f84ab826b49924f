"""CPU oracle for the evolution-strategies hot path  --  TEST INFRASTRUCTURE ONLY.

This module is a plain-numpy (fp32, step by step) restatement of what the reference
(nnaisense/evotorch @ cebcac4f, mounted read-only at /root/reference while developing)
computes on the per-generation path of its distribution-based searchers.  It exists so that
the CUDA kernels behind ``include/evok.h`` can be checked on machines where the reference
itself is not present (the GPU box).  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it; the product
package ``evotorch_b200`` never does.

Pinning: every function below is checked against outputs of the *real* reference, generated
in the build container by ``tests/golden/gen_golden.py`` (which imports /root/reference/src
through the ray/gymnasium import stubs) and committed as ``tests/golden/*.npz``; see
``tests/test_oracle_golden.py``.  It also reproduces the known-answer vectors of the
reference's own unit tests (tests/test_ranking.py:24-50, tests/test_optimizers.py:46-112,
tests/test_tools_misc.py:697-744).

All citations are ``path:line`` relative to /root/reference/src/evotorch.
"""

from __future__ import annotations

import math
from typing import Optional

import numpy as np

F32 = np.float32


def _f32(x) -> np.ndarray:
    return np.asarray(x, dtype=F32)


# --------------------------------------------------------------------------------------
# Ranking  (tools/ranking.py)
# --------------------------------------------------------------------------------------


def argsort_for_ranking(f: np.ndarray, higher_is_better: bool) -> np.ndarray:
    """`x.argsort(descending=not higher_is_better)` (tools/ranking.py:49,77,116) with the
    tie-break the new engine defines: a STABLE sort, i.e. equal fitnesses keep ascending index
    order in both directions (this is what torch.argsort(..., stable=True) returns; the
    reference's unstable default only differs on ties, see SURVEY.md section 7.2).
    -0.0 and +0.0 compare equal, NaN sorts as the largest value (torch semantics)."""
    f = _f32(f).reshape(-1)
    if higher_is_better:
        # ascending, stable; NaN last
        return np.argsort(f, kind="stable").astype(np.int64)
    # descending, stable: NaN (the largest value, above +inf) first, then by decreasing value; ties keep ascending index.
    nan = np.isnan(f)
    idx_nan = np.flatnonzero(nan)
    idx_rest = np.flatnonzero(~nan)
    order_rest = idx_rest[np.argsort(-f[idx_rest].astype(np.float64), kind="stable")]
    return np.concatenate([idx_nan, order_rest]).astype(np.int64)


def rank_centered(f, higher_is_better: bool) -> np.ndarray:
    """tools/ranking.py:24-53: w[idx[p]] = fp32(p)/(n-1) - 0.5, worst first."""
    f = _f32(f).reshape(-1)
    n = len(f)
    idx = argsort_for_ranking(f, higher_is_better)
    table = np.arange(n, dtype=F32) / F32(n - 1) - F32(0.5)
    out = np.empty(n, dtype=F32)
    out[idx] = table
    return out


def rank_linear(f, higher_is_better: bool) -> np.ndarray:
    """tools/ranking.py:56-81: like centered without the -0.5 shift."""
    f = _f32(f).reshape(-1)
    n = len(f)
    idx = argsort_for_ranking(f, higher_is_better)
    table = np.arange(n, dtype=F32) / F32(n - 1)
    out = np.empty(n, dtype=F32)
    out[idx] = table
    return out


def nes_utility_table(n: int) -> np.ndarray:
    """tools/ranking.py:107-114: u_p = max(0, ln(n/2+1) - ln(n-p)), p = 0 (worst) .. n-1 (best), fp32."""
    N = F32(n)
    incr = np.arange(n, dtype=F32)
    u = np.log(N / F32(2.0) + F32(1.0), dtype=F32) - np.log(N - incr, dtype=F32)
    return np.maximum(F32(0), u).astype(F32)


def rank_nes(f, higher_is_better: bool) -> np.ndarray:
    """tools/ranking.py:84-124: utils = u[ranks]; utils /= sum(utils); utils -= 1/n."""
    f = _f32(f).reshape(-1)
    n = len(f)
    idx = argsort_for_ranking(f, higher_is_better)
    ranks = np.empty(n, dtype=np.int64)
    ranks[idx] = np.arange(n, dtype=np.int64)
    utils = nes_utility_table(n)[ranks]
    utils = utils / np.sum(utils, dtype=F32)
    utils = utils - F32(1.0) / F32(n)
    return utils.astype(F32)


def rank_normalized(f, higher_is_better: bool) -> np.ndarray:
    """tools/ranking.py:127-160: (g - mean g)/std(g), unbiased std, g = f or -f."""
    g = _f32(f).reshape(-1)
    if not higher_is_better:
        g = -g
    mean = np.mean(g, dtype=F32)
    std = np.std(g.astype(np.float64), ddof=1).astype(F32)
    return ((g - mean) / std).astype(F32)


def rank_raw(f, higher_is_better: bool) -> np.ndarray:
    """tools/ranking.py:163-183."""
    g = _f32(f).reshape(-1)
    return g if higher_is_better else -g


RANKERS = {
    "centered": rank_centered,
    "linear": rank_linear,
    "nes": rank_nes,
    "normalized": rank_normalized,
    "raw": rank_raw,
}


def rank(f, ranking_method: str, higher_is_better: bool) -> np.ndarray:
    """tools/ranking.py:189-216 (KeyError on unknown method, like the reference's dict lookup)."""
    return RANKERS[ranking_method](f, higher_is_better)


# --------------------------------------------------------------------------------------
# Sampling layout (tools/misc.py:1663-1755) -- the RNG stream itself is not restated:
# given the standard-normal draws Z the reference places them like this.
# --------------------------------------------------------------------------------------


def population_from_normals(Z, mu, sigma, symmetric: bool) -> np.ndarray:
    """tools/misc.py:1731-1749.  symmetric: Z has N/2 rows; rows 2k / 2k+1 of the result are
    (Z_k * sigma) + mu and ((-Z_k) * sigma) + mu (separately rounded multiply then add).
    non-symmetric: Z has N rows; X = Z * sigma + mu."""
    Z = _f32(Z)
    mu = _f32(mu)
    sigma = _f32(sigma)
    if symmetric:
        K, D = Z.shape
        out = np.empty((2 * K, D), dtype=F32)
        out[0::2] = Z
        out[1::2] = -Z
    else:
        out = Z.copy()
    out = out * sigma
    out = out + mu
    return out.astype(F32)


# --------------------------------------------------------------------------------------
# Objective functions used by the benchmark configs
# --------------------------------------------------------------------------------------


def rastrigin(X) -> np.ndarray:
    """/root/reference/README.md:86-89: A*n + sum(x^2 - A*cos(2*pi*x)), A = 10.  Evaluated in
    float64 and rounded once: the oracle value for the fused evaluation kernel (which uses a
    different summation order and cos implementation than torch; compare with tolerance)."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[-1]
    return (10.0 * n + np.sum(X * X - 10.0 * np.cos(2.0 * math.pi * X), axis=-1)).astype(F32)


def sphere(X) -> np.ndarray:
    """sum(x^2) (reference tests/test_examples.py uses it as the smoke objective)."""
    X = np.asarray(X, dtype=np.float64)
    return np.sum(X * X, axis=-1).astype(F32)


# --------------------------------------------------------------------------------------
# Gradients  (distributions.py)
# --------------------------------------------------------------------------------------


def _colsum_weighted(w: np.ndarray, M: np.ndarray) -> np.ndarray:
    """total(dot(w, M)) of the reference = sum over rows of w_i * M_i (tools/misc.py:1089-1110).
    Accumulated in float64 and rounded once, so it is the *reference value* both the reference's
    fp32 result and the kernels' fp32 result are close to."""
    return (w.astype(np.float64)[:, None] * M.astype(np.float64)).sum(axis=0).astype(F32)


def _divide_grad(grad: np.ndarray, weights: np.ndarray, option: Optional[str]) -> np.ndarray:
    """distributions.py:517-536."""
    if option is None:
        return grad
    n = len(weights)
    if option == "num_solutions":
        return (grad / F32(n)).astype(F32)
    if option == "num_directions":
        return (grad / F32(n // 2)).astype(F32)
    if option == "total_weight":
        return (grad / np.sum(np.abs(weights), dtype=F32)).astype(F32)
    if option == "weight_stdev":
        return (grad / np.std(weights.astype(np.float64), ddof=1).astype(F32)).astype(F32)
    raise ValueError(f"unrecognized divide option {option!r}")


def grad_separable(X, w, mu, sigma, ranking_used: Optional[str], divide_mu_by=None, divide_sigma_by=None) -> dict:
    """SeparableGaussian._compute_gradients, distributions.py:548-579 (non-symmetric PGPE)."""
    X, w, mu, sigma = _f32(X), _f32(w), _f32(mu), _f32(sigma)
    eps = X - mu
    if ranking_used not in ("centered", "normalized"):
        w = (w - np.mean(w, dtype=F32)).astype(F32)
    gmu = _divide_grad(_colsum_weighted(w, eps), w, divide_mu_by)
    gsig = _divide_grad(_colsum_weighted(w, ((eps**2) - (sigma**2)) / sigma), w, divide_sigma_by)
    return {"mu": gmu, "sigma": gsig}


def grad_symmetric(X, w, mu, sigma, ranking_used: Optional[str], divide_mu_by=None, divide_sigma_by=None) -> dict:
    """SymmetricSeparableGaussian._compute_gradients, distributions.py:708-773."""
    X, w, mu, sigma = _f32(X), _f32(w), _f32(mu), _f32(sigma)
    if ranking_used not in ("centered", "normalized"):
        w = (w - np.mean(w, dtype=F32)).astype(F32)
    eps = X[0::2] - mu
    fdplus, fdminus = w[0::2], w[1::2]
    a = ((fdplus - fdminus) / F32(2)).astype(F32)
    b = ((fdplus + fdminus) / F32(2)).astype(F32)
    gmu = _divide_grad(_colsum_weighted(a, eps), w, divide_mu_by)
    gsig = _divide_grad(_colsum_weighted(b, ((eps**2) - (sigma**2)) / sigma), w, divide_sigma_by)
    return {"mu": gmu, "sigma": gsig}


def grad_parenthood(X, w, mu, sigma, parenthood_ratio: float) -> dict:
    """_compute_gradients_via_parenthood_ratio, distributions.py:538-546 (CEM): the
    floor(N*ratio) rows with the largest weights; mean(elites)-mu, std(elites, unbiased)-sigma.
    Tie-break among equal weights: stable descending (ascending index), as for ranking."""
    X, w, mu, sigma = _f32(X), _f32(w), _f32(mu), _f32(sigma)
    n = X.shape[0]
    num_elites = int(math.floor(n * parenthood_ratio))
    elite_idx = argsort_for_ranking(w, higher_is_better=False)[:num_elites]
    elites = X[elite_idx].astype(np.float64)
    return {
        "mu": (elites.mean(axis=0).astype(F32) - mu).astype(F32),
        "sigma": (elites.std(axis=0, ddof=1).astype(F32) - sigma).astype(F32),
        "elite_indices": elite_idx,
    }


def grad_exp_separable(X, w, mu, sigma, ranking_used: Optional[str]) -> dict:
    """ExpSeparableGaussian._compute_gradients, distributions.py:783-793 (SNES)."""
    X, w, mu, sigma = _f32(X), _f32(w), _f32(mu), _f32(sigma)
    if ranking_used != "nes":
        w = (w / np.sum(np.abs(w), dtype=F32)).astype(F32)
    eps = X - mu
    raw = eps / sigma
    return {"mu": _colsum_weighted(w, eps), "sigma": _colsum_weighted(w, (raw**2) - F32(1))}


def grad_exp_gaussian(X, w, mu, A_inv, ranking_used: Optional[str]) -> dict:
    """ExpGaussian._compute_gradients, distributions.py:963-989 (XNES): z = A^-1 (x - mu);
    d = sum w z; M = sum w (z z^T - I)."""
    X, w, mu, A_inv = _f32(X), _f32(w), _f32(mu), _f32(A_inv)
    Zl = (A_inv.astype(np.float64) @ (X - mu).astype(np.float64).T).T
    if ranking_used not in ("centered", "normalized"):
        w = (w - np.mean(w, dtype=F32)).astype(F32)
    w64 = w.astype(np.float64)
    d = (w64[:, None] * Zl).sum(axis=0)
    M = (Zl.T * w64) @ Zl - w64.sum() * np.eye(Zl.shape[1])
    return {"d": d.astype(F32), "M": M.astype(F32)}


# --------------------------------------------------------------------------------------
# Optimizers (optimizers.py) and parameter updates (distributions.py, tools/misc.py)
# --------------------------------------------------------------------------------------


class ClipUp:
    """optimizers.py:231-357.  v <- clip_norm(m*v + lr*g/||g||, max_speed); ascent returns v."""

    def __init__(self, solution_length: int, stepsize: float, momentum: float = 0.9, max_speed: Optional[float] = None):
        self.stepsize = float(stepsize)
        self.momentum = float(momentum)
        self.max_speed = 2.0 * self.stepsize if max_speed is None else float(max_speed)  # :274-275
        self.velocity = np.zeros(int(solution_length), dtype=F32)

    def ascent(self, g) -> np.ndarray:
        g = _f32(g)
        gnorm = np.sqrt(np.sum(g.astype(np.float64) ** 2)).astype(F32)
        grad = (g / gnorm) * F32(self.stepsize)  # :348
        v = (F32(self.momentum) * self.velocity) + grad  # :350
        vnorm = np.sqrt(np.sum(v.astype(np.float64) ** 2)).astype(F32)
        if vnorm > self.max_speed:  # :313
            v = v * (F32(self.max_speed) / vnorm)
        self.velocity = v.astype(F32)
        return self.velocity.copy()


class Adam:
    """optimizers.py:101-165 + TorchOptimizer.ascent :60-91: torch.optim.Adam on a zeroed dummy
    parameter whose .grad is the ascent direction g; ascent = -param after step() =
    lr * m_hat / (sqrt(v_hat) + eps) with torch defaults lr=1e-3, betas=(0.9, 0.999), eps=1e-8."""

    def __init__(self, solution_length: int, stepsize: Optional[float] = None, beta1=None, beta2=None, epsilon=None):
        self.lr = 1e-3 if stepsize is None else float(stepsize)
        self.b1 = 0.9 if beta1 is None else float(beta1)
        self.b2 = 0.999 if beta2 is None else float(beta2)
        self.eps = 1e-8 if epsilon is None else float(epsilon)
        self.m = np.zeros(int(solution_length), dtype=F32)
        self.v = np.zeros(int(solution_length), dtype=F32)
        self.t = 0

    def ascent(self, g) -> np.ndarray:
        g = _f32(g)
        self.t += 1
        self.m = (F32(self.b1) * self.m + F32(1 - self.b1) * g).astype(F32)
        self.v = (F32(self.b2) * self.v + F32(1 - self.b2) * g * g).astype(F32)
        bc1 = 1 - self.b1**self.t
        bc2 = 1 - self.b2**self.t
        step_size = self.lr / bc1
        denom = (np.sqrt(self.v) / F32(math.sqrt(bc2))) + F32(self.eps)
        return (F32(step_size) * (self.m / denom)).astype(F32)


class SGD:
    """optimizers.py:168-228: torch.optim.SGD (momentum buffer b <- mom*b + g, first step b = g;
    no dampening/nesterov by default); ascent = lr * b."""

    def __init__(self, solution_length: int, stepsize: float, momentum: Optional[float] = None):
        self.lr = float(stepsize)
        self.momentum = 0.0 if momentum is None else float(momentum)
        self.buf = None
        self.n = int(solution_length)

    def ascent(self, g) -> np.ndarray:
        g = _f32(g)
        if self.momentum != 0.0:
            if self.buf is None:
                self.buf = g.copy()
            else:
                self.buf = (F32(self.momentum) * self.buf + g).astype(F32)
            d = self.buf
        else:
            d = g
        return (F32(self.lr) * d).astype(F32)


def modify_tensor(original, target, lb=None, ub=None, max_change=None) -> np.ndarray:
    """tools/misc.py:711-816: clamp `target` into [max(lb, o-|o|c), min(ub, o+|o|c)]."""
    original, target = _f32(original), _f32(target)
    if lb is None and ub is None and max_change is None:
        return target
    lo = _f32(-np.inf if lb is None else lb)
    hi = _f32(np.inf if ub is None else ub)
    if max_change is not None:
        allowed = np.abs(original) * _f32(max_change)
        lo = np.maximum(lo, original - allowed)
        hi = np.minimum(hi, original + allowed)
    return np.minimum(np.maximum(target, lo), hi).astype(F32)


def follow_gradient(g, learning_rate=None, optimizer=None) -> np.ndarray:
    """Distribution._follow_gradient, distributions.py:372-392."""
    g = _f32(g)
    if learning_rate is None and optimizer is None:
        return g
    if optimizer is None:
        return (F32(learning_rate) * g).astype(F32)
    if learning_rate is None:
        return optimizer.ascent(g)
    raise ValueError("both learning_rate and optimizer given")


def update_separable(mu, sigma, grads, lr_mu=None, lr_sigma=None, opt_mu=None) -> tuple:
    """SeparableGaussian.update_parameters, distributions.py:581-596."""
    mu, sigma = _f32(mu), _f32(sigma)
    new_mu = mu + follow_gradient(grads["mu"], lr_mu, opt_mu)
    new_sigma = sigma + follow_gradient(grads["sigma"], lr_sigma, None)
    return new_mu.astype(F32), new_sigma.astype(F32)


def update_exp_separable(mu, sigma, grads, lr_mu=None, lr_sigma=None, opt_mu=None) -> tuple:
    """ExpSeparableGaussian.update_parameters, distributions.py:795-810 (SNES)."""
    mu, sigma = _f32(mu), _f32(sigma)
    new_mu = mu + follow_gradient(grads["mu"], lr_mu, opt_mu)
    new_sigma = sigma * np.exp(F32(0.5) * follow_gradient(grads["sigma"], lr_sigma, None), dtype=F32)
    return new_mu.astype(F32), new_sigma.astype(F32)


def update_distribution(
    mu, sigma, grads, *, exp_sigma: bool, lr_mu, lr_sigma, opt_mu=None, stdev_min=None, stdev_max=None, stdev_max_change=None
) -> tuple:
    """GaussianSearchAlgorithm._update_distribution, algorithms/distributed/gaussian.py:369-419:
    parameter update followed by the controlled-sigma clamp against the pre-update sigma."""
    lr_mu_eff = None if opt_mu is not None else lr_mu
    if exp_sigma:
        new_mu, new_sigma = update_exp_separable(mu, sigma, grads, lr_mu_eff, lr_sigma, opt_mu)
    else:
        new_mu, new_sigma = update_separable(mu, sigma, grads, lr_mu_eff, lr_sigma, opt_mu)
    if stdev_min is not None or stdev_max is not None or stdev_max_change is not None:
        new_sigma = modify_tensor(sigma, new_sigma, lb=stdev_min, ub=stdev_max, max_change=stdev_max_change)
    return new_mu, new_sigma


# --------------------------------------------------------------------------------------
# One generation of the Gaussian searchers, given the population (gaussian.py:351-367)
# --------------------------------------------------------------------------------------

ALGO_DEFAULTS = {
    # name: (symmetric, exp_sigma, ranking, divide_by, default optimizer)
    "pgpe": dict(symmetric=True, exp_sigma=False, ranking="centered", divide="num_directions"),
    "pgpe_nonsym": dict(symmetric=False, exp_sigma=False, ranking="centered", divide="num_solutions"),
    "snes": dict(symmetric=False, exp_sigma=True, ranking="nes", divide=None),
}


def gaussian_generation_update(algo: str, X, f, mu, sigma, sense: str, *, lr_mu, lr_sigma, opt_mu=None,
                               ranking: Optional[str] = "__default__", stdev_min=None, stdev_max=None,
                               stdev_max_change=None, parenthood_ratio=None) -> dict:
    """What `_step_non_distributed` does with the stored population of the previous generation
    (gaussian.py:357-366): rank -> gradients -> update (-> clamp).  Returns weights, gradients and the
    new (mu, sigma)."""
    hib = {"max": True, "min": False}[sense]
    if algo == "cem":
        method = None if ranking == "__default__" else ranking
        w = rank(f, "raw" if method is None else method, hib)
        grads = grad_parenthood(X, w, mu, sigma, parenthood_ratio)
        new_mu, new_sigma = update_distribution(mu, sigma, grads, exp_sigma=False, lr_mu=1.0, lr_sigma=1.0,
                                                stdev_min=stdev_min, stdev_max=stdev_max,
                                                stdev_max_change=stdev_max_change)
        return {"weights": w, "grads": grads, "mu": new_mu, "sigma": new_sigma}
    cfg = ALGO_DEFAULTS[algo]
    method = cfg["ranking"] if ranking == "__default__" else ranking
    w = rank(f, "raw" if method is None else method, hib)
    if algo == "pgpe":
        grads = grad_symmetric(X, w, mu, sigma, method, cfg["divide"], cfg["divide"])
    elif algo == "pgpe_nonsym":
        grads = grad_separable(X, w, mu, sigma, method, cfg["divide"], cfg["divide"])
    else:
        grads = grad_exp_separable(X, w, mu, sigma, method)
    new_mu, new_sigma = update_distribution(mu, sigma, grads, exp_sigma=cfg["exp_sigma"], lr_mu=lr_mu,
                                            lr_sigma=lr_sigma, opt_mu=opt_mu, stdev_min=stdev_min,
                                            stdev_max=stdev_max, stdev_max_change=stdev_max_change)
    return {"weights": w, "grads": grads, "mu": new_mu, "sigma": new_sigma}


# --------------------------------------------------------------------------------------
# XNES update (distributions.py:991-1016)
# --------------------------------------------------------------------------------------


def _expm(M64: np.ndarray) -> np.ndarray:
    """Matrix exponential in float64 (scaling and squaring with a Taylor core)."""
    n = M64.shape[0]
    norm = np.linalg.norm(M64, 1)
    s = max(0, int(math.ceil(math.log2(norm))) + 1) if norm > 0 else 0
    A = M64 / (2.0**s)
    E = np.eye(n)
    term = np.eye(n)
    for k in range(1, 25):
        term = term @ A / k
        E = E + term
    for _ in range(s):
        E = E @ E
    return E


def update_exp_gaussian(mu, A, A_inv, grads, lr_mu, lr_sigma, opt_mu=None) -> tuple:
    """ExpGaussian.update_parameters, distributions.py:991-1016: mu' = mu + A (follow d);
    A' = A expm(0.5 lr M); A_inv' = expm(-0.5 lr M) A_inv."""
    mu, A, A_inv = _f32(mu), _f32(A), _f32(A_inv)
    upd_d = follow_gradient(grads["d"], None if opt_mu is not None else lr_mu, opt_mu)
    upd_M = follow_gradient(grads["M"], lr_sigma, None).astype(np.float64)
    new_mu = mu + (A.astype(np.float64) @ upd_d.astype(np.float64)).astype(F32)
    new_A = A.astype(np.float64) @ _expm(0.5 * upd_M)
    new_A_inv = _expm(-0.5 * upd_M) @ A_inv.astype(np.float64)
    return new_mu.astype(F32), new_A.astype(F32), new_A_inv.astype(F32)


# --------------------------------------------------------------------------------------
# CMA-ES (algorithms/cmaes.py)
# --------------------------------------------------------------------------------------


class CMAESState:
    """Hyper-parameters and state of the reference CMAES for the non-separable case
    (algorithms/cmaes.py:279-385), computed in float64 then held as python floats / fp32 arrays.
    The `*_ratio` arguments scale the default hyper-parameters as the reference's do (each one before the
    defaults that depend on it); `stdev_min` / `stdev_max` bound sqrt(diag(C)) * sigma (`cmaes_limit_stdev`)."""

    def __init__(self, d: int, popsize: int, stdev_init: float, center, active: bool = True, c_m: float = 1.0,
                 csa_squared: bool = False, limit_C_decomposition: bool = True, c_sigma_ratio: float = 1.0,
                 damp_sigma_ratio: float = 1.0, c_c_ratio: float = 1.0, c_1_ratio: float = 1.0, c_mu_ratio: float = 1.0,
                 stdev_min: Optional[float] = None, stdev_max: Optional[float] = None):
        self.d = int(d)
        self.popsize = int(popsize)
        self.mu_count = int(math.floor(popsize / 2))
        self.m = _f32(center).copy()
        self.sigma = F32(stdev_init)
        self.C = np.eye(d, dtype=F32)
        self.A = np.eye(d, dtype=F32)
        # raw weights :302 (computed in fp32 by the reference: make_tensor of a float64 -> problem dtype)
        raw = (np.log((popsize + 1) / 2) - np.log(np.arange(popsize, dtype=np.float64) + 1)).astype(F32)
        pos, neg = raw[: self.mu_count], raw[self.mu_count:]
        self.mu_eff = F32(np.sum(pos, dtype=F32) ** 2 / np.sum(pos**2, dtype=F32))
        mu_eff = float(self.mu_eff)
        self.c_m = c_m
        self.active = active
        self.csa_squared = csa_squared
        self.stdev_min, self.stdev_max = stdev_min, stdev_max
        self.c_sigma = c_sigma_ratio * ((mu_eff + 2.0) / (d + mu_eff + 3))
        self.damp_sigma = damp_sigma_ratio * (1 + 2 * max(0.0, math.sqrt((mu_eff - 1) / (d + 1)) - 1) + self.c_sigma)
        self.c_c = c_c_ratio * ((4 + mu_eff / d) / (d + (4 + 2 * mu_eff / d)))
        self.c_1 = c_1_ratio * (min(1, popsize / 6) * 2 / ((d + 1.3) ** 2.0 + mu_eff))
        self.c_mu = c_mu_ratio * min(1 - self.c_1, 2 * ((0.25 + mu_eff - 2 + (1 / mu_eff)) / ((d + 2) ** 2.0 + mu_eff)))
        self.variance_discount_sigma = math.sqrt(self.c_sigma * (2 - self.c_sigma) * mu_eff)
        self.variance_discount_c = math.sqrt(self.c_c * (2 - self.c_c) * mu_eff)
        pos = pos / np.sum(pos, dtype=F32)
        if active:
            mu_eff_neg = float(np.sum(neg, dtype=F32) ** 2 / np.sum(neg**2, dtype=F32))
            alpha = min(1 + self.c_1 / self.c_mu, 1 + 2 * mu_eff_neg / (mu_eff + 2),
                        (1 - self.c_mu - self.c_1) / (d * self.c_mu))
            neg = F32(alpha) * neg / np.sum(np.abs(neg), dtype=F32)
        else:
            neg = np.zeros_like(neg)
        self.weights = np.concatenate([pos, neg]).astype(F32)
        self.p_sigma = np.zeros(d, dtype=F32)
        self.p_c = np.zeros(d, dtype=F32)
        self.unbiased_expectation = math.sqrt(d) * (1 - (1 / (4 * d)) + 1 / (21 * d**2))
        if limit_C_decomposition:
            b = 10 * d * (self.c_1 + self.c_mu)
            b = b if abs(b) >= 1e-8 else (1e-8 if b >= 0 else -1e-8)
            self.decompose_C_freq = max(1, int(math.floor(1 / b)))
        else:
            self.decompose_C_freq = 1
        self.steps = 0


def cmaes_sample(state: CMAESState, Z) -> tuple:
    """sample_distribution, cmaes.py:408-430: ys = (A zs^T)^T, xs = m + sigma ys."""
    Z = _f32(Z)
    Y = (state.A.astype(np.float64) @ Z.astype(np.float64).T).T.astype(F32)
    X = (state.m[None, :] + state.sigma * Y).astype(F32)
    return Y, X


def cmaes_assign_weights(state: CMAESState, f, sense: str) -> np.ndarray:
    """get_population_weights, cmaes.py:432-452: argsort best-first (SolutionBatch.argsort,
    core.py:3827-3844), inverse permutation, gather.  Stable tie-break."""
    f = _f32(f)
    # best first: for "min" ascending f, for "max" descending f
    order = argsort_for_ranking(f, higher_is_better=(sense == "min"))
    ranks = np.empty(len(f), dtype=np.int64)
    ranks[order] = np.arange(len(f))
    return state.weights[ranks]


def cmaes_recombine(state: CMAESState, Z, Y, assigned_weights) -> tuple:
    """update_m :454-481, the sums only: local = sum_i w_i z_i and shaped = sum_i w_i y_i over the mu best (the top-mu
    weights are exactly the positive ones: stable order by weight desc), in float64."""
    Z, Y, aw = _f32(Z), _f32(Y), _f32(assigned_weights)
    top = np.argsort(-aw.astype(np.float64), kind="stable")[: state.mu_count]
    tw = aw[top].astype(np.float64)
    local_disp = (tw[:, None] * Z[top].astype(np.float64)).sum(axis=0)
    shaped_disp = (tw[:, None] * Y[top].astype(np.float64)).sum(axis=0)
    return local_disp, shaped_disp


def cmaes_h_sig(state: CMAESState, pnorm: float) -> tuple:
    """_h_sig :31-46 from ||p_sigma|| after this generation's update and the generation counter BEFORE its increment.
    Returns (h_sig, margin): margin = |lhs - rhs| / rhs of the comparison lhs < rhs that decides it."""
    d = state.d
    squared_sum = pnorm**2 / (1 - (1 - state.c_sigma) ** (2 * state.steps + 1))
    lhs, rhs = (squared_sum / d) - 1, 1 + 4.0 / (d + 1)
    return (1.0 if lhs < rhs else 0.0), abs(lhs - rhs) / rhs


def cmaes_vector_step(state: CMAESState, local_disp, shaped_disp) -> float:
    """update_m (with the OLD sigma), update_p_sigma, update_sigma, _h_sig and update_p_c (:454-517, :31-46): the work of
    evok_cmaes_vector_update.  Updates the state; returns h_sig."""
    d = state.d
    state.m = (state.m + F32(state.c_m) * state.sigma * np.asarray(shaped_disp).astype(F32)).astype(F32)
    # update_p_sigma :483-490
    state.p_sigma = (F32(1 - state.c_sigma) * state.p_sigma
                     + F32(state.variance_discount_sigma) * np.asarray(local_disp).astype(F32)).astype(F32)
    # update_sigma :492-507
    pnorm = float(np.sqrt(np.sum(state.p_sigma.astype(np.float64) ** 2)))
    if state.csa_squared:
        expo = (pnorm**2 / d - 1) / 2
    else:
        expo = pnorm / state.unbiased_expectation - 1
    state.sigma = F32(state.sigma * np.exp(F32((state.c_sigma / state.damp_sigma) * expo)))
    h_sig, _ = cmaes_h_sig(state, pnorm)
    # update_p_c :509-517
    state.p_c = (F32(1 - state.c_c) * state.p_c
                 + F32(h_sig * state.variance_discount_c) * np.asarray(shaped_disp).astype(F32)).astype(F32)
    return h_sig


def cmaes_covariance_coefficients(state: CMAESState, h_sig: float) -> tuple:
    """update_C :537-541: (c1a, weighted_pc).  The update C <- C + c1a (pc pc^T - C) + c_mu (S - sum(w) C), pc =
    weighted_pc p_c, is k1 C + k0 S + k2 p_c p_c^T with the three coefficients of `cmaes_k`."""
    c1a = state.c_1 * (1 - (1 - h_sig**2) * state.c_c * (2 - state.c_c))
    weighted_pc = (state.c_1 / (c1a + 1e-23)) ** 0.5
    return c1a, weighted_pc


def cmaes_k(state: CMAESState, h_sig: float) -> tuple:
    """(k0, k1, k2) = (c_mu, 1 - c1a - c_mu sum(w), c1a weighted_pc^2): what evok_cmaes_vector_update writes to `k_out`."""
    c1a, weighted_pc = cmaes_covariance_coefficients(state, h_sig)
    return state.c_mu, 1 - c1a - state.c_mu * float(np.sum(state.weights, dtype=F32)), c1a * weighted_pc**2


def cmaes_active_weights(state: CMAESState, Z, assigned_weights) -> np.ndarray:
    """update_C :531-535: w_i > 0 ? w_i : d w_i / ||z_i||^2 with active weights, w unchanged otherwise (float64)."""
    w = _f32(assigned_weights).astype(np.float64)
    if state.active:
        zn2 = (_f32(Z).astype(np.float64) ** 2).sum(axis=1)
        w = np.where(w > 0, w, state.d * w / zn2)
    return w


def cmaes_covariance_update(state: CMAESState, Y, w, c1a: float, weighted_pc: float) -> None:
    """update_C :543-553: the rank-1 and rank-mu update of C with the (active-reweighted) weights `w`."""
    pc = weighted_pc * state.p_c.astype(np.float64)
    C64 = state.C.astype(np.float64)
    r1 = c1a * (np.outer(pc, pc) - C64)
    Y64 = _f32(Y).astype(np.float64)
    rmu = state.c_mu * ((Y64.T * w) @ Y64 - float(np.sum(state.weights, dtype=F32)) * C64)
    state.C = (C64 + r1 + rmu).astype(F32)


def cmaes_limit_stdev(state: CMAESState) -> None:
    """_limit_stdev :49-79, non-separable: only the diagonal of C is rewritten, to (clamp(sigma sqrt(C_ii), lo, hi) / sigma)^2."""
    if state.stdev_min is None and state.stdev_max is None:
        return
    sigma = np.float64(state.sigma)
    stdevs = np.clip(sigma * np.sqrt(np.diag(state.C).astype(np.float64)), state.stdev_min, state.stdev_max)
    C = state.C.copy()
    np.fill_diagonal(C, ((stdevs / sigma) ** 2).astype(F32))
    state.C = C


def cmaes_decomposition_due(state: CMAESState) -> bool:
    """decompose_C :555-565: A is refactorised on the generations where (steps + 1) % decompose_C_freq == 0."""
    return (state.steps + 1) % state.decompose_C_freq == 0


def cmaes_decompose(state: CMAESState) -> None:
    state.A = np.linalg.cholesky(state.C.astype(np.float64)).astype(F32)


def cmaes_update(state: CMAESState, Z, Y, assigned_weights) -> None:
    """cmaes.py:454-606 (_step after evaluation), non-separable branch; float64 accumulation,
    fp32 state."""
    local_disp, shaped_disp = cmaes_recombine(state, Z, Y, assigned_weights)
    h_sig = cmaes_vector_step(state, local_disp, shaped_disp)
    c1a, weighted_pc = cmaes_covariance_coefficients(state, h_sig)
    cmaes_covariance_update(state, Y, cmaes_active_weights(state, Z, assigned_weights), c1a, weighted_pc)
    cmaes_limit_stdev(state)
    if cmaes_decomposition_due(state):
        cmaes_decompose(state)
    state.steps += 1


# --------------------------------------------------------------------------------------
# Batched flat-parameter policy forward (neuroevolution/net/vecrl.py:1240-1279,
# net/functional.py:118-200): row = [W1 (H x I, row-major), b1 (H), W2 (O x H), b2 (O)]
# --------------------------------------------------------------------------------------


def mlp_policy_forward(params, obs, n_in: int, n_hidden: int, n_out: int, activation: str = "tanh") -> np.ndarray:
    params = np.asarray(params, dtype=np.float64)
    obs = np.asarray(obs, dtype=np.float64)
    N = params.shape[0]
    o = 0
    W1 = params[:, o:o + n_hidden * n_in].reshape(N, n_hidden, n_in); o += n_hidden * n_in
    b1 = params[:, o:o + n_hidden]; o += n_hidden
    W2 = params[:, o:o + n_out * n_hidden].reshape(N, n_out, n_hidden); o += n_out * n_hidden
    b2 = params[:, o:o + n_out]; o += n_out
    assert o == params.shape[1]
    h = np.einsum("nhi,ni->nh", W1, obs) + b1
    if activation == "tanh":
        h = np.tanh(h)
    elif activation == "relu":
        h = np.maximum(h, 0)
    elif activation != "none":
        raise ValueError(activation)
    return (np.einsum("noh,nh->no", W2, h) + b2).astype(F32)


# --------------------------------------------------------------------------------------
# The kernels' Philox4x32-10 sampler (include/evok.h, evok_sample_eval).  Not part of the reference
# (which draws from torch's generator, tools/misc.py:1739): this restates the NEW engine's documented
# counter mapping so the GPU tests can check it (geometry / shard independence, known-answer vectors of
# Random123's philox4x32-10).
# --------------------------------------------------------------------------------------

_PHILOX_M0, _PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_PHILOX_W0, _PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0: int, k1: int) -> tuple:
    """Vectorised Philox4x32-10 (Salmon, Moraes, Dror, Shaw; SC'11).  Counters are uint32 arrays, keys python ints."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _MASK32 for c in (c0, c1, c2, c3))
    for _ in range(10):
        p0 = _PHILOX_M0 * c0
        p1 = _PHILOX_M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK32
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0 = (k0 + _PHILOX_W0) & 0xFFFFFFFF
        k1 = (k1 + _PHILOX_W1) & 0xFFFFFFFF
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def _box_muller(a: np.ndarray, b: np.ndarray) -> tuple:
    u1 = a.astype(np.float64) * 2.0**-32 + 2.0**-33
    th = 2.0 * math.pi * (b.astype(np.float64) * 2.0**-32 + 2.0**-33)
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(th), r * np.sin(th)


def philox_normals(seed: int, stream_id: int, units: np.ndarray, D: int) -> np.ndarray:
    """Standard normals z[unit, column] of the kernels' sampler (float64; the kernels use fast fp32 intrinsics, so
    compare with ~1e-5 absolute tolerance).  counter = (column // 4, unit_lo, unit_hi, stream_id_lo),
    key = (seed_lo, seed_hi ^ stream_id_hi); outputs (x, y) -> columns 4q, 4q+1 and (z, w) -> 4q+2, 4q+3."""
    units = np.asarray(units, dtype=np.uint64)
    nq = (D + 3) // 4
    q = np.arange(nq, dtype=np.uint64)
    U, Q = np.meshgrid(units, q, indexing="ij")
    k0 = seed & 0xFFFFFFFF
    k1 = ((seed >> 32) ^ (stream_id >> 32)) & 0xFFFFFFFF
    x, y, z, w = philox4x32_10(Q, U & _MASK32, U >> np.uint64(32), np.full_like(Q, stream_id & 0xFFFFFFFF), k0, k1)
    z0, z1 = _box_muller(x, y)
    z2, z3 = _box_muller(z, w)
    out = np.stack([z0, z1, z2, z3], axis=-1).reshape(len(units), nq * 4)
    return out[:, :D]


def philox_population(mu, sigma, n_rows: int, symmetric: bool, seed: int, stream_id: int, row0: int = 0) -> np.ndarray:
    """Population rows [row0, row0 + n_rows) written by evok_sample_eval (float64 math, rounded to fp32)."""
    mu = np.asarray(mu, dtype=np.float64)
    sigma = np.asarray(sigma, dtype=np.float64)
    D = len(mu)
    if symmetric:
        units = np.arange(row0 // 2, (row0 + n_rows) // 2)
        Z = philox_normals(seed, stream_id, units, D)
        X = np.empty((n_rows, D))
        X[0::2] = mu + sigma * Z
        X[1::2] = mu - sigma * Z
    else:
        Z = philox_normals(seed, stream_id, np.arange(row0, row0 + n_rows), D)
        X = mu + sigma * Z
    return X.astype(F32)
