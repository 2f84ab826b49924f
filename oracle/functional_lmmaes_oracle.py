"""Float64 numpy restatement of LM-MA-ES (Loshchilov, Glasmachers & Beyer, IEEE TEVC 23(2), 2019) for one search, in the paper's
form: the ask makes k = min(t, m) serial row reductions per row, and the tell undoes them one vector at a time.

    state = init(center, sigma, popsize=None, num_vectors=None, maximize=False)
    X = ask(state, Z)                 # Z (popsize, D) standard normal
    state = tell(state, X, f)         # a new dict; the input is left unchanged

The state is a dict: y (D,), sigma, p_sigma (D,), M (m, D), t and the constants.
"""

from __future__ import annotations

import math

import numpy as np


def constants(d: int, popsize=None, num_vectors=None) -> dict:
    lam = 4 + int(math.floor(3 * math.log(d))) if popsize is None else int(popsize)
    m = 4 + int(math.floor(3 * math.log(d))) if num_vectors is None else int(num_vectors)
    mu = lam // 2
    raw = np.log(mu + 0.5) - np.log(np.arange(1, mu + 1))
    w = raw / raw.sum()
    j = np.arange(m)
    return dict(popsize=lam, mu=mu, weights=w, mu_eff=1.0 / np.sum(w**2), num_vectors=m, c_sigma=2.0 * lam / d,
                c_d=1.0 / (1.5**j * d), c_c=lam / (4.0**j * d))


def init(center, sigma, popsize=None, num_vectors=None, maximize=False) -> dict:
    y = np.asarray(center, np.float64).copy()
    c = constants(y.size, popsize, num_vectors)
    return dict(y=y, sigma=float(sigma), p_sigma=np.zeros(y.size), M=np.zeros((c["num_vectors"], y.size)), t=0, maximize=bool(maximize), **c)


def _k(state) -> int:
    return min(state["t"], state["num_vectors"])


def steps(state, Z) -> np.ndarray:
    """d_i of every row: z_i, then for j = 1..k: d <- (1 - c_d,j) d + c_d,j M_j (M_j^T d)."""
    D = np.array(Z, np.float64, copy=True)
    for j in range(_k(state)):
        mj, c = state["M"][j], state["c_d"][j]
        D = (1 - c) * D + c * np.outer(D @ mj, mj)
    return D


def ask(state, Z) -> np.ndarray:
    return state["y"] + state["sigma"] * steps(state, Z)


def recover(state, D) -> np.ndarray:
    """The z of steps d: for j = k..1, v <- (v - kappa_j M_j (M_j^T v)) / (1 - c_d,j), kappa_j = c_d,j / ((1 - c_d,j) + c_d,j |M_j|^2)."""
    V = np.array(D, np.float64, copy=True)
    for j in reversed(range(_k(state))):
        mj, c = state["M"][j], state["c_d"][j]
        kappa = c / ((1 - c) + c * (mj @ mj))
        V = (V - kappa * np.outer(V @ mj, mj)) / (1 - c)
    return V


def rank_weights(state, f) -> np.ndarray:
    """w_1..w_mu on the best mu rows, 0 on the rest: the order of the functional CMA-ES tell, a stable sort (ties by row) that
    takes NaN as the largest value, ascending to minimise and descending to maximise."""
    f = np.asarray(f, np.float64)
    nan = np.isnan(f)
    if state["maximize"]:
        order = np.lexsort((np.arange(f.size), np.where(nan, 0.0, -f), ~nan))
    else:
        order = np.lexsort((np.arange(f.size), np.where(nan, 0.0, f), nan))
    w = np.zeros(f.size)
    w[order[: state["mu"]]] = state["weights"]
    return w


def tell(state, X, f) -> dict:
    s = dict(state)
    w = rank_weights(state, f)
    D = (np.asarray(X, np.float64) - state["y"]) / state["sigma"]
    Z = recover(state, D)
    S_z, S_d = w @ Z, w @ D
    cs, mu_eff = state["c_sigma"], state["mu_eff"]
    s["p_sigma"] = (1 - cs) * state["p_sigma"] + math.sqrt(mu_eff * cs * (2 - cs)) * S_z
    cc = state["c_c"]
    s["M"] = (1 - cc)[:, None] * state["M"] + np.sqrt(mu_eff * cc * (2 - cc))[:, None] * S_z[None, :]
    s["y"] = state["y"] + state["sigma"] * S_d
    s["sigma"] = state["sigma"] * math.exp((cs / 2) * (s["p_sigma"] @ s["p_sigma"] / state["y"].size - 1))
    s["t"] = state["t"] + 1
    return s
