"""The restart stage of the functional CMA-ES families (evok_cma_restart_batched, funcrestarts._restart_torch), restated per item
in float64 numpy: best ever, the tol_fun history, the seven stop criteria and the re-initialisation.

The new centre of a restarted item b is lb + (ub - lb) * u with u_j = uniform24 of word j & 3 of Philox4x32-10 at counter
(j >> 2, 0, 0xFF000000, b) under key (seed, stream 0) on the kernels (`reset_uniforms`), computed in float32 without fused
multiply-adds there (`centre`); the torch path takes u from torch.rand.
"""

from __future__ import annotations

import math

import numpy as np

from .es_oracle import philox4x32_10
from .noise_oracle import _key, uniform24

RESET_TAG = 0xFF000000
BITS = ("tol_fun", "tol_x", "tol_x_up", "max_condition", "min_fitness_stdev", "max_generations", "non_finite")


def reset_uniforms(seed: int, B: int, D: int) -> np.ndarray:
    """[B, D] float64: the u of every item's reset draw on the kernels."""
    nq = (D + 3) // 4
    Bq, Q = np.meshgrid(np.arange(B, dtype=np.uint64), np.arange(nq, dtype=np.uint64), indexing="ij")
    words = philox4x32_10(Q, np.zeros_like(Q), np.full_like(Q, RESET_TAG), Bq & np.uint64(0xFFFFFFFF), *_key(seed, 0))
    return np.stack([uniform24(w) for w in words], axis=-1).reshape(B, nq * 4)[:, :D]


def centre(lb, ub, u, float32: bool) -> np.ndarray:
    """lb + (ub - lb) * u, each operation rounded to float32 (the kernels) or in float64."""
    if float32:
        lb, ub, u = (np.asarray(t, dtype=np.float32) for t in (lb, ub, u))
        return (lb + (ub - lb) * u).astype(np.float64)
    return np.asarray(lb, np.float64) + (np.asarray(ub, np.float64) - np.asarray(lb, np.float64)) * np.asarray(u, np.float64)


def _nanmax(v, init):
    v = np.asarray(v, np.float64)
    v = v[~np.isnan(v)]
    return max(init, float(v.max())) if v.size else init


def _nanmin(v, init):
    v = np.asarray(v, np.float64)
    v = v[~np.isnan(v)]
    return min(init, float(v.min())) if v.size else init


def restart_item(*, f, x_rows, gen, sigma, m, p_sigma, p_c, c_diag, r_diag, separable, history, best_x, best_f, num_restarts, sigma0, lb, ub,
                 thresholds, maximize, u, float32) -> dict:
    """One item after its update.  f [N]; x_rows [N, D] (the told rows); gen: its counter after the update; c_diag = diag C;
    r_diag: diag A (full) or C (separable); history [H]; thresholds: 6 floats or None (ops.RESTART_CRITERIA order); u [D].
    Returns the item's new fields and `flags`, `reset` (bool) and `centre` (the new centre when reset)."""
    f = np.asarray(f, np.float64)
    N, H = f.size, len(history)
    history = np.array(history, np.float64)
    best_x, best_f = np.array(best_x, np.float64), float(best_f)
    fin = np.isfinite(f)
    g_best, idx = math.nan, -1
    for i in range(N):  # the lower row wins ties
        if fin[i] and (idx < 0 or (f[i] > g_best if maximize else f[i] < g_best)):
            g_best, idx = float(f[i]), i
    if idx >= 0 and (g_best > best_f if maximize else g_best < best_f):
        best_x, best_f = np.array(x_rows[idx], np.float64), g_best
    if gen >= 1:
        history[(gen - 1) % H] = g_best
    tol_fun, tol_x, tol_x_up, max_cond, min_std, max_gen = thresholds
    c_diag, r_diag = np.asarray(c_diag, np.float64), np.asarray(r_diag, np.float64)
    max_pc = _nanmax(np.abs(np.asarray(p_c, np.float64)), 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        max_sd = _nanmax(np.sqrt(c_diag), 0.0)
        q = _nanmax(r_diag, -math.inf) / _nanmin(r_diag, math.inf)
    flags = 0
    if tol_fun is not None and gen >= H and fin.all() and np.isfinite(history).all():
        if max(f.max(), history.max()) - min(f.min(), history.min()) < tol_fun:
            flags |= 1
    if tol_x is not None and sigma * max(max_pc, max_sd) < tol_x * sigma0:
        flags |= 2
    if tol_x_up is not None and sigma * max_sd > tol_x_up * sigma0:
        flags |= 4
    if max_cond is not None and (q if separable else q * q) > max_cond:
        flags |= 8
    if min_std is not None and N > 1 and np.std(f, ddof=1) < min_std:
        flags |= 16
    if max_gen is not None and gen >= max_gen:
        flags |= 32
    state = np.concatenate([np.atleast_1d(np.asarray(t, np.float64)) for t in (m, p_sigma, p_c, c_diag)])
    if not (sigma > 0) or not math.isfinite(sigma) or not np.isfinite(state).all():
        flags |= 64
    out = dict(best_x=best_x, best_f=best_f, history=history, flags=flags, reset=flags != 0, gen=gen, num_restarts=num_restarts, centre=None)
    if flags:
        out.update(centre=centre(lb, ub, u, float32), gen=0, history=np.full(H, math.nan), num_restarts=num_restarts + 1)
    return out


def constructed_items(separable: bool, maximize: bool, D: int = 5, N: int = 8, seed: int = 0) -> dict:
    """Ten items (float32 values as float64) built so that each criterion fires on one of them and not on item 0:
    0 nothing (a tie for the best row: rows 2 and 5), 1 tol_x, 2 tol_x_up, 3 max_condition, 4 min_fitness_stdev, 5 max_generations,
    6 non-finite, 7 tol_fun (and min_fitness_stdev), 8 NaN and inf fitnesses with an earlier best ever that stays, 9 no finite
    fitness.  Full family: C = diag(c_diag), A = diag(r_diag)."""
    rng = np.random.default_rng(seed)
    B, H = 10, 10 + math.ceil(30 * D / N)
    sgn = -1.0 if maximize else 1.0
    c = dict(B=B, D=D, N=N, H=H, separable=separable, maximize=maximize, thresholds=(1e-12, 1e-12, 1e4, 1e14, 1e-6, 50.0))
    c["f"] = rng.normal(size=(B, N)) * 3
    c["X"] = rng.normal(size=(B, N, D))
    c["gen"] = np.full(B, 5, np.int64)
    c["sigma"] = np.full(B, 0.5)
    c["sigma0"] = rng.uniform(0.5, 2.0, B)
    c["m"] = rng.normal(size=(B, D))
    c["p_sigma"] = rng.normal(size=(B, D)) * 0.1
    c["p_c"] = rng.normal(size=(B, D)) * 0.1
    c["c_diag"] = rng.uniform(0.5, 2.0, (B, D))
    c["history"] = rng.normal(size=(B, H))
    c["best_x"] = np.full((B, D), math.nan)
    c["best_f"] = np.full(B, sgn * math.inf)
    c["num_restarts"] = rng.integers(0, 4, B)
    c["lb"] = rng.uniform(-6.0, -1.0, (B, D))
    c["ub"] = c["lb"] + rng.uniform(0.5, 8.0, (B, D))
    c["f"][0, [2, 5]] = sgn * -10.0
    c["sigma"][1] = 1e-14
    c["sigma"][2] = 1e5
    c["c_diag"][3, 0] = 1e-15 if separable else 1e-16
    c["f"][4] = 3.0
    c["gen"][5] = 60
    c["p_c"][6, 1] = math.nan
    c["gen"][7] = H + 3
    c["history"][7] = 2.0
    c["f"][7] = 2.0
    c["f"][8, :3] = (math.nan, math.inf, -math.inf)
    c["best_f"][8] = sgn * -100.0
    c["best_x"][8] = 1.0
    c["f"][9] = math.nan
    for k in ("f", "X", "sigma", "sigma0", "m", "p_sigma", "p_c", "c_diag", "history", "best_x", "best_f", "lb", "ub"):
        c[k] = np.asarray(c[k], np.float32).astype(np.float64)
    c["r_diag"] = c["c_diag"] if separable else np.sqrt(c["c_diag"]).astype(np.float32).astype(np.float64)
    return c


def expected(c: dict, u: np.ndarray, float32: bool) -> list:
    """restart_item for every item of a `constructed_items` case (x_rows: c["X"], or c["rows"] when the case carries them)."""
    rows = c.get("rows", c["X"])
    return [restart_item(f=c["f"][b], x_rows=rows[b], gen=int(c["gen"][b]), sigma=float(c["sigma"][b]), m=c["m"][b], p_sigma=c["p_sigma"][b],
                         p_c=c["p_c"][b], c_diag=c["c_diag"][b], r_diag=c["r_diag"][b], separable=c["separable"], history=c["history"][b],
                         best_x=c["best_x"][b], best_f=c["best_f"][b], num_restarts=int(c["num_restarts"][b]), sigma0=float(c["sigma0"][b]),
                         lb=c["lb"][b], ub=c["ub"][b], thresholds=c["thresholds"], maximize=c["maximize"], u=u[b], float32=float32)
            for b in range(c["B"])]


DESIGNED = {1: 2, 2: 4, 3: 8, 4: 16, 5: 32, 6: 64, 7: 1}  # item -> a bit its construction must raise
