"""Functional LM-MA-ES: `lmmaes(...) -> LMMAESState`, `lmmaes_ask(state)`, `lmmaes_ask_and_evaluate(state, ...)`,
`lmmaes_tell(state, values, evals)`.

The limited-memory matrix adaptation evolution strategy (Loshchilov, Glasmachers & Beyer, "Large Scale Black-box Optimization by
Limited-Memory Matrix Adaptation", IEEE TEVC 23(2), 2019), with explicit state and extra leftmost batch dimensions: every batch
item is an independent search with its own centre y, step size, path p_sigma and m direction vectors M; the population size,
weights and learning rates are shared.  In place of a D x D covariance each item keeps the m ~ 4 + 3 ln D vectors, so state and
work per sample are O(m D), and unlike separable CMA-ES the search learns rotations.

At generation t, k = min(t, m) vectors are in use.  A row's step is z after k steps d <- (1 - c_d,j) d + c_d,j M_j (M_j^T d); the
tell recovers z from the values (so repaired or injected solutions are legal) and updates p_sigma, every M_j, y and sigma.  The
state also holds G = M M^T, which lets every stage work in the coefficient form d_i = alpha z_i + sum_j beta_ij M_j.

On CUDA float32 a generation of ALL items is a fixed number of launches per item chunk of 65535 items (ops.lmmaes_ask_batched /
lmmaes_tell_batched): the ask is a Gram pass P = M Z^T over z rebuilt from Philox, the coefficient recursion and the pass that
writes x (only the last at t = 0); the tell is the rank table, a pass over the rows with non-zero weight, the recovery, the update
of M, p_sigma, y with G of the new M, and sigma.  Nothing is read back to the host.  The kernels take popsize <= 128 and
num_vectors <= 64.  Anywhere else the same algorithm runs as batched torch ops in the same coefficient form.
"""

from __future__ import annotations

import math
from typing import Callable, NamedTuple, Optional

import torch

from ... import ops
from .funccmaes import _assigned_weights
from .fused import ask_and_evaluate_keyed
from .misc import draw_philox_seed, on_kernels


class LMMAESHyperparameters(NamedTuple):
    popsize: int  # lambda
    mu: int
    weights: torch.Tensor  # (popsize,): w_1 .. w_mu, then zeros
    mu_eff: float
    num_vectors: int  # m
    c_sigma: float
    c_d: tuple  # m floats, c_d,j = 1 / (1.5^(j-1) D)
    c_c: tuple  # m floats, c_c,j = lambda / (4^(j-1) D)

    def consts(self) -> tuple:
        """The constants of the kernels: (c_sigma, mu_eff, c_d[m], c_c[m])."""
        return (self.c_sigma, self.mu_eff) + self.c_d + self.c_c


def lmmaes_hyperparameters(d: int, popsize: Optional[int] = None, num_vectors: Optional[int] = None, *, dtype=torch.float32,
                           device="cpu") -> LMMAESHyperparameters:
    """The shared constants of an LM-MA-ES search of solution length d; ValueError where they are not defined."""
    default = 4 + int(math.floor(3 * math.log(d)))
    lam = default if popsize is None else int(popsize)
    m = default if num_vectors is None else int(num_vectors)
    if lam < 2:
        raise ValueError(f"`popsize` must be at least 2, got {lam}")
    if m < 1:
        raise ValueError(f"`num_vectors` must be at least 1, got {m}")
    c_sigma = 2.0 * lam / d
    if c_sigma >= 1:
        raise ValueError(f"LM-MA-ES needs c_sigma = 2 popsize / D < 1: with popsize {lam} the solution length must be at least {2 * lam + 1}, "
                         f"got {d}")
    mu = lam // 2
    raw = [math.log(mu + 0.5) - math.log(i) for i in range(1, mu + 1)]
    total = sum(raw)
    w = [r / total for r in raw]
    mu_eff = 1.0 / sum(x * x for x in w)
    weights = torch.zeros(lam, dtype=dtype, device=device)
    weights[:mu] = torch.tensor(w, dtype=torch.float64).to(dtype)
    c_d = tuple(1.0 / (1.5**j * d) for j in range(m))
    c_c = tuple(lam / (4.0**j * d) for j in range(m))
    return LMMAESHyperparameters(lam, mu, weights, mu_eff, m, c_sigma, c_d, c_c)


class LMMAESState(NamedTuple):
    center: torch.Tensor  # (..., D), y
    sigma: torch.Tensor  # (...)
    p_sigma: torch.Tensor  # (..., D)
    M: torch.Tensor  # (..., m, D), the direction vectors
    G: torch.Tensor  # (..., m, m), M M^T
    generation: int  # t, shared by every item
    hyperparameters: LMMAESHyperparameters
    maximize: bool

    @property
    def popsize(self) -> int:
        return self.hyperparameters.popsize

    @property
    def num_vectors(self) -> int:
        return self.hyperparameters.num_vectors


def lmmaes(*, center_init, stdev_init, objective_sense: str, popsize: Optional[int] = None, num_vectors: Optional[int] = None) -> LMMAESState:
    """Initial state.  `center_init` (..., D); `stdev_init` a scalar or a tensor of batch shape; the batch shape of the search is
    their broadcast.  popsize and num_vectors default to 4 + floor(3 ln D).  ValueError for an objective sense other than "min" /
    "max", popsize < 2, num_vectors < 1, D <= 2 popsize (c_sigma = 2 popsize / D must be below 1) and, for a state on the kernels
    (float32 CUDA), popsize > 128 or num_vectors > 64."""
    if objective_sense not in ("min", "max"):
        raise ValueError(f"`objective_sense` was expected as 'min' or 'max', but it was received as {objective_sense!r}")
    center_init = torch.as_tensor(center_init)
    if not center_init.is_floating_point():
        center_init = center_init.to(torch.get_default_dtype())
    if center_init.ndim < 1 or center_init.shape[-1] == 0:
        raise ValueError(f"`center_init` was expected with shape (..., D), D >= 1; got {tuple(center_init.shape)}")
    dtype, device, d = center_init.dtype, center_init.device, center_init.shape[-1]
    sigma = torch.as_tensor(stdev_init, dtype=dtype, device=device)
    batch = tuple(torch.broadcast_shapes(center_init.shape[:-1], sigma.shape))
    hp = lmmaes_hyperparameters(d, popsize, num_vectors, dtype=dtype, device=device)
    if on_kernels(center_init):
        if hp.popsize > ops.LMMAES_MAX_POPSIZE:
            raise ValueError(f"the LM-MA-ES kernels take popsize <= {ops.LMMAES_MAX_POPSIZE}, got {hp.popsize}")
        if hp.num_vectors > ops.LMMAES_MAX_VECTORS:
            raise ValueError(f"the LM-MA-ES kernels take num_vectors <= {ops.LMMAES_MAX_VECTORS}, got {hp.num_vectors}")
    m = hp.num_vectors
    return LMMAESState(
        center=center_init.expand(batch + (d,)).contiguous().clone(),
        sigma=sigma.expand(batch).contiguous().clone(),
        p_sigma=torch.zeros(batch + (d,), dtype=dtype, device=device),
        M=torch.zeros(batch + (m, d), dtype=dtype, device=device),
        G=torch.zeros(batch + (m, m), dtype=dtype, device=device),
        generation=0,
        hyperparameters=hp,
        maximize=(objective_sense == "max"),
    )


def _items(state: LMMAESState) -> tuple:
    """(batch shape, number of items B, D) of a state."""
    batch, d = tuple(state.center.shape[:-1]), state.center.shape[-1]
    return batch, math.prod(batch), d


def _flat(state: LMMAESState, B: int, d: int) -> tuple:
    m = state.num_vectors
    return (state.center.reshape(B, d), state.sigma.reshape(B), state.p_sigma.reshape(B, d), state.M.reshape(B, m, d),
            state.G.reshape(B, m, m))


def _ask_torch(state: LMMAESState, z: torch.Tensor) -> torch.Tensor:
    """The population (B, popsize, D) of the steps z (B, popsize, D), in the coefficient form: P = M_k z^T, then for j < k
    s = alpha P_j + beta G_j, alpha, beta *= (1 - c_d,j), beta_j += c_d,j s; x = y + sigma (alpha z + beta M_k)."""
    hp = state.hyperparameters
    B, n, d = z.shape
    y, sigma, _, M, G = _flat(state, B, d)
    k = min(state.generation, hp.num_vectors)
    Mk, Gk = M[:, :k], G[:, :k, :k]
    P = torch.einsum("bkd,bnd->bkn", Mk, z)
    alpha = 1.0
    beta = torch.zeros(B, n, k, dtype=z.dtype, device=z.device)
    for j in range(k):
        s = alpha * P[:, j, :] + torch.einsum("bnl,bl->bn", beta, Gk[:, :, j])
        alpha *= 1 - hp.c_d[j]
        beta = beta * (1 - hp.c_d[j])
        beta[:, :, j] += hp.c_d[j] * s
    dsteps = alpha * z + torch.einsum("bnk,bkd->bnd", beta, Mk)
    return y[:, None, :] + sigma[:, None, None] * dsteps


def _ask(state: LMMAESState) -> tuple:
    """(`lmmaes_ask`'s population, the Philox seed of its draw on the kernels (item b on stream b), None elsewhere)."""
    batch, B, d = _items(state)
    n = state.popsize
    y, sigma, _, M, G = _flat(state, B, d)
    if on_kernels(y, sigma, M, G):
        seed = draw_philox_seed()
        k = min(state.generation, state.num_vectors)
        x = ops.lmmaes_ask_batched(y, sigma, M, G, k, state.hyperparameters.consts(), n, seed=seed)
        return x.view(batch + (n, d)), seed
    z = torch.randn(B, n, d, dtype=y.dtype, device=y.device)
    return _ask_torch(state, z).view(batch + (n, d)), None


def lmmaes_ask(state: LMMAESState) -> torch.Tensor:
    """A population per item, (..., popsize, D): row i of item b is y_b + sigma_b d_i, d_i the step of z_i ~ N(0, I) through the
    item's first min(t, m) vectors.  On the kernels z_i of item b is the row `ops.sample_batched` draws on Philox stream b."""
    return _ask(state)[0]


def lmmaes_ask_and_evaluate(state: LMMAESState, *, objective: Callable) -> tuple:
    """`lmmaes_ask` and the fitnesses of the population: (values (..., popsize, D), evals (..., popsize)).  The population is
    stored.  With the state on the kernels, an objective with `evaluate_batched` (the objectives of evotorch_b200.objectives and
    every FusedObjective, transformed and noisy ones included) evaluates all items in one call, keyed with the ask's Philox seed,
    so a noisy objective gets the noise of the draw and per-item data gives item b its own data.  Otherwise this is `lmmaes_ask`
    followed by `objective(values)`.  An objective whose data has a batch shape must have the state's batch shape."""
    return ask_and_evaluate_keyed(lambda: _ask(state), _items(state)[0], objective, "LM-MA-ES")


def _recovery_torch(state: LMMAESState, d_steps: torch.Tensor) -> tuple:
    """(a, gamma (B, n, k)) with z_i = a d_i + sum_j gamma_ij M_j: the tell's recovery in the coefficient form, from Q = M_k d^T,
    for j = k-1 .. 0: u = a Q_j + gamma G_j, a, gamma /= (1 - c_d,j), gamma_j -= kappa_j u / (1 - c_d,j)."""
    hp = state.hyperparameters
    B, n, d = d_steps.shape
    _, _, _, M, G = _flat(state, B, d)
    k = min(state.generation, hp.num_vectors)
    Q = torch.einsum("bkd,bnd->bkn", M[:, :k], d_steps)
    a = 1.0
    gamma = torch.zeros(B, n, k, dtype=d_steps.dtype, device=d_steps.device)
    for j in reversed(range(k)):
        f = 1 - hp.c_d[j]
        kappa = hp.c_d[j] / (f + hp.c_d[j] * G[:, j, j])
        u = a * Q[:, j, :] + torch.einsum("bnl,bl->bn", gamma, G[:, :k, j])
        a = a / f
        gamma = gamma / f
        gamma[:, :, j] -= (kappa[:, None] * u) / f
    return a, gamma


def _recovered_steps(state: LMMAESState, values: torch.Tensor) -> torch.Tensor:
    """The z (B, popsize, D) that the tell recovers from `values`: the inverse of the ask's steps, up to rounding."""
    _, B, d = _items(state)
    y, sigma, _, M, _ = _flat(state, B, d)
    d_steps = (values.reshape(B, -1, d) - y[:, None, :]) / sigma[:, None, None]
    a, gamma = _recovery_torch(state, d_steps)
    k = gamma.shape[-1]
    return a * d_steps + torch.einsum("bnk,bkd->bnd", gamma, M[:, :k])


def lmmaes_tell(state: LMMAESState, values: torch.Tensor, evals: torch.Tensor) -> LMMAESState:
    """The next state, given a population `values` (..., popsize, D) and its fitnesses `evals` (..., popsize).  The steps are
    recovered from the values, so repaired or injected solutions are legal.  The state passed in is left unchanged."""
    batch, B, d = _items(state)
    hp = state.hyperparameters
    n, m = hp.popsize, hp.num_vectors
    y = state.center
    values = torch.as_tensor(values, dtype=y.dtype, device=y.device)
    evals = torch.as_tensor(evals, dtype=y.dtype, device=y.device)
    if tuple(values.shape) != batch + (n, d):
        raise ValueError(f"`values` was expected with shape {batch + (n, d)}, got {tuple(values.shape)}")
    if tuple(evals.shape) != batch + (n,):
        raise ValueError(f"`evals` was expected with shape {batch + (n,)}, got {tuple(evals.shape)}")
    x, f = values.reshape(B, n, d), evals.reshape(B, n)
    k = min(state.generation, m)
    y0, sigma, p_sigma, M, G = _flat(state, B, d)
    if on_kernels(y0, x, f):
        aw = ops.rank_table_batched(f, state.maximize, hp.weights)
        y1, sigma1, p1, M1, G1 = ops.lmmaes_tell_batched(x.contiguous(), aw, y0.contiguous(), sigma.contiguous(), p_sigma.contiguous(),
                                                         M.contiguous(), G.contiguous(), k, hp.consts())
    else:
        y1, sigma1, p1, M1, G1 = _tell_torch(state, hp, x, f, y0, sigma, p_sigma, M)
    return state._replace(center=y1.view(batch + (d,)), sigma=sigma1.view(batch), p_sigma=p1.view(batch + (d,)), M=M1.view(batch + (m, d)),
                          G=G1.view(batch + (m, m)), generation=state.generation + 1)


def _tell_torch(state, hp, x, f, y, sigma, p_sigma, M) -> tuple:
    """The tell as batched torch ops, in the coefficient form of the kernels."""
    d = x.shape[-1]
    aw = _assigned_weights(f, state.maximize, hp.weights)
    d_steps = (x - y[:, None, :]) / sigma[:, None, None]
    S_d = torch.einsum("bn,bnd->bd", aw, d_steps)
    a, gamma = _recovery_torch(state, d_steps)
    k = gamma.shape[-1]
    S_z = a * S_d + torch.einsum("bk,bkd->bd", torch.einsum("bn,bnk->bk", aw, gamma), M[:, :k])
    cs = hp.c_sigma
    p_sigma = (1 - cs) * p_sigma + math.sqrt(hp.mu_eff * cs * (2 - cs)) * S_z
    cc = torch.tensor(hp.c_c, dtype=x.dtype, device=x.device)
    M = (1 - cc)[None, :, None] * M + torch.sqrt(hp.mu_eff * cc * (2 - cc))[None, :, None] * S_z[:, None, :]
    y = y + sigma[:, None] * S_d
    sigma = sigma * torch.exp((cs / 2) * (torch.sum(p_sigma * p_sigma, dim=-1) / d - 1))
    return y, sigma, p_sigma, M, M @ M.mT
