"""Functional XNES: `xnes(...) -> XNESState`, `xnes_ask(state)`, `xnes_ask_and_evaluate(state, ...)`, `xnes_tell(state, values, evals)`.

Exponential natural evolution strategies (Glasmachers, Schaul, Yi, Wierstra & Schmidhuber, "Exponential Natural Evolution
Strategies", GECCO 2010), the algorithm of `algorithms.gaussian.XNES` (same defaults, utilities and update), with explicit state
and extra leftmost batch dimensions: every batch item is an independent search with its own centre mu and factor A (samples are
x = mu + A z) and A's inverse; the population size, learning rates and ranking are shared.

The tell recovers z = A_inv (x - mu) from the values, so repaired or injected solutions are legal, then with utilities w
    d = sum w_i z_i,  G = sum w_i z_i z_i^T - (sum w) I,  S = (eta_A / 2) G,
    mu' = mu + eta_mu A d,  A' = A expm(S),  A_inv' = expm(-S) A_inv.

On CUDA float32 a generation of ALL items is a fixed number of launches per item chunk of 65535 items: the ask is the batched
Philox sampler and the batched GEMM x = mu + z A^T (the draw path of `cmaes_ask`), the tell is the rank, the centring of the
utilities and one CTA per item (ops.xnes_tell_batched) that forms d and S in shared memory and applies the update through the
exponential pair expm(+-S) - I.  Nothing is read back to the host.  The kernels take D <= ops.XNES_MAX_D (96).  Anywhere else
(CPU, float64) the same algorithm runs as batched torch ops with `torch.matrix_exp`.
"""

from __future__ import annotations

import math
from typing import Callable, NamedTuple, Optional

import torch

from ... import ops
from .fused import ask_and_evaluate_keyed
from .misc import draw_philox_seed, on_kernels


class XNESState(NamedTuple):
    center: torch.Tensor  # (..., D), mu
    A: torch.Tensor  # (..., D, D): samples are mu + A z
    A_inv: torch.Tensor  # (..., D, D)
    popsize: int
    center_learning_rate: float  # eta_mu
    stdev_learning_rate: float  # eta_A
    ranking_method: str
    maximize: bool


def default_popsize(d: int) -> int:
    """4 + floor(3 ln D), the population size of XNES and SNES."""
    return 4 + int(math.floor(3 * math.log(d)))


def rank_rows(f: torch.Tensor, method: str, maximize: bool) -> torch.Tensor:
    """The utilities of `tools.ranking.rank` for every row of f (B, n) at once, as torch ops (a stable sort, best last)."""
    B, n = f.shape
    g = f if maximize else -f
    if method == "raw":
        return g
    if method == "normalized":
        return (g - g.mean(-1, keepdim=True)) / g.std(-1, keepdim=True)
    steps = torch.arange(n, dtype=f.dtype, device=f.device)
    if method == "centered":
        table = steps / (n - 1) - 0.5
    elif method == "linear":
        table = steps / (n - 1)
    elif method == "nes":
        nf = torch.tensor(n, dtype=f.dtype, device=f.device)
        table = torch.clamp_min(torch.log(nf / 2.0 + 1.0) - torch.log(nf - steps), 0.0)
    else:
        raise ValueError(f"unknown ranking method {method!r}; expected one of {sorted(ops.RANK_IDS)}")
    order = torch.argsort(f, dim=-1, descending=not maximize, stable=True)
    out = torch.empty_like(f).scatter_(-1, order, table.expand(B, n).contiguous())
    if method == "nes":
        out = out / out.sum(-1, keepdim=True) - 1 / nf
    return out


def check_ranking_method(method: str) -> str:
    if method not in ops.RANK_IDS:
        raise ValueError(f"unknown ranking method {method!r}; expected one of {sorted(ops.RANK_IDS)}")
    return str(method)


def xnes(*, center_init, stdev_init, objective_sense: str, popsize: Optional[int] = None, center_learning_rate: Optional[float] = None,
         stdev_learning_rate: Optional[float] = None, scale_learning_rate: bool = True, ranking_method: str = "nes") -> XNESState:
    """Initial state.  `center_init` (..., D); `stdev_init` a scalar, (D,) or (..., D): A_0 = diag(stdev_init); the batch shape of
    the search is the broadcast of the centre's batch dimensions and stdev_init's.  Defaults are those of `XNES`: popsize
    4 + floor(3 ln D), eta_mu = 1, eta_A = 0.6 (3 + ln D) / (D sqrt D), a given stdev_learning_rate multiplied by that default when
    `scale_learning_rate`.  ValueError for an objective sense other than "min" / "max", popsize < 2, an unknown ranking method and,
    for a state on the kernels (float32 CUDA), D > ops.XNES_MAX_D."""
    if objective_sense not in ("min", "max"):
        raise ValueError(f"`objective_sense` was expected as 'min' or 'max', but it was received as {objective_sense!r}")
    center_init = torch.as_tensor(center_init)
    if not center_init.is_floating_point():
        center_init = center_init.to(torch.get_default_dtype())
    if center_init.ndim < 1 or center_init.shape[-1] == 0:
        raise ValueError(f"`center_init` was expected with shape (..., D), D >= 1; got {tuple(center_init.shape)}")
    dtype, device, d = center_init.dtype, center_init.device, center_init.shape[-1]
    stdev = torch.as_tensor(stdev_init, dtype=dtype, device=device)
    if stdev.ndim == 0:
        stdev = stdev.expand(d)
    if stdev.shape[-1] != d:
        raise ValueError(f"`stdev_init` was expected as a scalar, ({d},) or (..., {d}); got {tuple(stdev.shape)}")
    popsize = default_popsize(d) if popsize is None else int(popsize)
    if popsize < 2:
        raise ValueError(f"`popsize` must be at least 2, got {popsize}")
    if on_kernels(center_init) and d > ops.XNES_MAX_D:
        raise ValueError(f"the XNES kernels take D <= {ops.XNES_MAX_D}, got {d}: use `cmaes` or `lmmaes` for longer solutions on the GPU, "
                         "or run XNES in float64, where it takes the torch path")
    default_lr = 0.6 * (3 + math.log(d)) / (d * math.sqrt(d))
    if stdev_learning_rate is None:
        lr_A = default_lr
    else:
        lr_A = float(stdev_learning_rate) * (default_lr if scale_learning_rate else 1.0)
    batch = tuple(torch.broadcast_shapes(center_init.shape[:-1], stdev.shape[:-1]))
    stdev = stdev.expand(batch + (d,))
    return XNESState(
        center=center_init.expand(batch + (d,)).contiguous().clone(),
        A=torch.diag_embed(stdev).contiguous(),
        A_inv=torch.diag_embed(1 / stdev).contiguous(),
        popsize=popsize,
        center_learning_rate=1.0 if center_learning_rate is None else float(center_learning_rate),
        stdev_learning_rate=lr_A,
        ranking_method=check_ranking_method(ranking_method),
        maximize=(objective_sense == "max"),
    )


def _items(state: XNESState) -> tuple:
    """(batch shape, number of items B, D) of a state; ValueError if A or A_inv does not match the centre."""
    batch, d = tuple(state.center.shape[:-1]), state.center.shape[-1]
    for name in ("A", "A_inv"):
        if tuple(getattr(state, name).shape) != batch + (d, d):
            raise ValueError(f"`{name}` was expected with shape {batch + (d, d)} (the centre's), got {tuple(getattr(state, name).shape)}")
    return batch, math.prod(batch), d


def _ask(state: XNESState) -> tuple:
    """(`xnes_ask`'s population, the Philox seed of its z on the kernels (item b on stream b), None elsewhere)."""
    batch, B, d = _items(state)
    n = state.popsize
    mu, A = state.center.reshape(B, d), state.A.reshape(B, d, d)
    if on_kernels(mu, A):
        z = torch.empty(B, n, d, dtype=torch.float32, device=mu.device)
        zero = torch.zeros(d, dtype=torch.float32, device=mu.device)
        seed = draw_philox_seed()
        ops.sample_batched(z, zero, zero + 1.0, symmetric=False, seed=seed)
        x = torch.empty_like(z)
        ops.gemm_nt_batched(z, A.contiguous(), torch.empty_like(z), out2=x, bias=mu.contiguous())
        return x.view(batch + (n, d)), seed
    z = torch.randn(B, n, d, dtype=mu.dtype, device=mu.device)
    return (mu[:, None, :] + z @ A.mT).view(batch + (n, d)), None


def xnes_ask(state: XNESState) -> torch.Tensor:
    """A population per item, (..., popsize, D): row i of item b is mu_b + A_b z_i, z_i ~ N(0, I).  On the kernels z is drawn as
    `cmaes_ask` draws it, item b on Philox stream b."""
    return _ask(state)[0]


def xnes_ask_and_evaluate(state: XNESState, *, objective: Callable) -> tuple:
    """`xnes_ask` and the fitnesses of the population: (values (..., popsize, D), evals (..., popsize)).  The population is stored.
    With the state on the kernels, an objective with `evaluate_batched` (the objectives of evotorch_b200.objectives and every
    FusedObjective, transformed and noisy ones included) evaluates all items in one call, keyed with the ask's Philox seed, so a
    noisy objective gets the noise of the draw and per-item data gives item b its own data.  Otherwise this is `xnes_ask`
    followed by `objective(values)`.  An objective whose data has a batch shape must have the state's batch shape."""
    return ask_and_evaluate_keyed(lambda: _ask(state), _items(state)[0], objective, "XNES")


def xnes_tell(state: XNESState, values: torch.Tensor, evals: torch.Tensor) -> XNESState:
    """The next state, given a population `values` (..., popsize, D) and its fitnesses `evals` (..., popsize).  The steps are
    recovered from the values, so repaired or injected solutions are legal.  The state passed in is left unchanged."""
    batch, B, d = _items(state)
    n = state.popsize
    mu = state.center
    values = torch.as_tensor(values, dtype=mu.dtype, device=mu.device)
    evals = torch.as_tensor(evals, dtype=mu.dtype, device=mu.device)
    if tuple(values.shape) != batch + (n, d):
        raise ValueError(f"`values` was expected with shape {batch + (n, d)}, got {tuple(values.shape)}")
    if tuple(evals.shape) != batch + (n,):
        raise ValueError(f"`evals` was expected with shape {batch + (n,)}, got {tuple(evals.shape)}")
    x, f = values.reshape(B, n, d), evals.reshape(B, n)
    mu, A, A_inv = mu.reshape(B, d), state.A.reshape(B, d, d), state.A_inv.reshape(B, d, d)
    if on_kernels(mu, A, A_inv, x, f):
        if d > ops.XNES_MAX_D:
            raise ValueError(f"the XNES kernels take D <= {ops.XNES_MAX_D}, got {d}: use `cmaes` or `lmmaes` for longer solutions on the "
                             "GPU, or run XNES in float64, where it takes the torch path")
        w = ops.rank_batched(f.contiguous(), state.ranking_method, state.maximize)
        if state.ranking_method not in ("centered", "normalized"):
            ops.weights_adjust_batched_(w, 1)  # w - mean(w)
        mu1, A1, A_inv1 = ops.xnes_tell_batched(x.contiguous(), w, mu.contiguous(), A.contiguous(), A_inv.contiguous(), state.center_learning_rate,
                                                state.stdev_learning_rate)
    else:
        mu1, A1, A_inv1 = _tell_torch(state, x, f, mu, A, A_inv)
    return state._replace(center=mu1.view(batch + (d,)), A=A1.view(batch + (d, d)), A_inv=A_inv1.view(batch + (d, d)))


def _tell_torch(state: XNESState, x, f, mu, A, A_inv) -> tuple:
    """The tell as batched torch ops, in the order of ExpGaussian._compute_gradients and update_parameters."""
    w = rank_rows(f, state.ranking_method, state.maximize)
    if state.ranking_method not in ("centered", "normalized"):
        w = w - w.mean(-1, keepdim=True)
    z = (x - mu[:, None, :]) @ A_inv.mT
    grad_d = torch.einsum("bn,bnd->bd", w, z)
    eye = torch.eye(mu.shape[-1], dtype=mu.dtype, device=mu.device)
    grad_M = (z.mT * w[:, None, :]) @ z - w.sum(-1)[:, None, None] * eye
    upd_d, upd_M = state.center_learning_rate * grad_d, state.stdev_learning_rate * grad_M
    mu = mu + (A @ upd_d[:, :, None])[:, :, 0]
    return mu, A @ torch.matrix_exp(0.5 * upd_M), torch.matrix_exp(-0.5 * upd_M) @ A_inv
