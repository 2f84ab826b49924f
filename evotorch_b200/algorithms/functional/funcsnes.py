"""Functional SNES: `snes(...) -> SNESState`, `snes_ask(state)`, `snes_ask_and_evaluate(state, ...)`, `snes_tell(state, values, evals)`.

Separable natural evolution strategies (Schaul, Glasmachers & Schmidhuber, "High Dimensions and Heavy Tails for Natural Evolution
Strategies", GECCO 2011), the algorithm of `algorithms.gaussian.SNES` (same defaults, utilities, exponential stdev update and
stdev bounds), with explicit state and extra leftmost batch dimensions: every batch item is an independent search with its own
centre and stdev vector; the population size, learning rates and ranking are shared.

With utilities w (divided by sum |w| unless the ranking is "nes") and eps_i = x_i - mu:
    grad_mu = sum w_i eps_i,  grad_sigma = sum w_i ((eps_i / sigma)^2 - 1),
    mu' = mu + eta_mu grad_mu (or the step of `optimizer`),  sigma' = sigma exp(eta_sigma grad_sigma / 2), clamped to the bounds.

On CUDA float32 a generation of ALL items is one launch per stage: sampling (with a fused objective, sample-and-evaluate), rank,
the division by sum |w|, the weighted sums (ops.grad_batched with GRAD_EXP; with `lazy=True` the population is not stored and
its rows are rebuilt from their Philox counters), the stdev update with its bounds, and the centre step.  Anywhere else the same
algorithm runs as batched torch ops.
"""

from __future__ import annotations

import math
from typing import Callable, NamedTuple, Optional, Union

import torch

from ... import ops
from ...tools import modify_tensor
from .funcpgpe import sample_separable
from .funcxnes import check_ranking_method, default_popsize, rank_rows
from .fused import LazyPopulation, ask_and_evaluate
from .misc import flat_items, get_functional_optimizer, on_kernels, vector_like_center


class SNESState(NamedTuple):
    center: torch.Tensor  # (..., D)
    stdev: torch.Tensor  # (..., D)
    optimizer: Optional[Union[str, tuple]]  # None: mu + eta_mu grad_mu
    optimizer_state: Optional[tuple]
    popsize: int
    center_learning_rate: float  # eta_mu
    stdev_learning_rate: float  # eta_sigma
    stdev_min: Optional[torch.Tensor]
    stdev_max: Optional[torch.Tensor]
    stdev_max_change: Optional[torch.Tensor]
    ranking_method: str
    maximize: bool


def snes(*, center_init, stdev_init, objective_sense: str, popsize: Optional[int] = None, center_learning_rate: Optional[float] = None,
         stdev_learning_rate: Optional[float] = None, scale_learning_rate: bool = True, ranking_method: str = "nes", optimizer=None,
         optimizer_config: Optional[dict] = None, stdev_min=None, stdev_max=None, stdev_max_change=None) -> SNESState:
    """Initial state.  `center_init` (..., D); `stdev_init` a scalar, (D,) or (..., D); the batch shape of the search is their
    broadcast.  Defaults are those of `SNES`: popsize 4 + floor(3 ln D), eta_mu = 1, eta_sigma = 0.2 (3 + ln D) / sqrt D, a given
    stdev_learning_rate multiplied by that default when `scale_learning_rate`.  `optimizer` ("clipup", "adam", "sgd" or a
    functional triple, configured by `optimizer_config`) follows grad_mu with step size eta_mu, as in `pgpe`.  The stdev bounds
    are scalars or (D,) / (..., D) tensors, applied against the stdev before each update.  ValueError for an objective sense other
    than "min" / "max", popsize < 2 and an unknown ranking method."""
    if objective_sense not in ("min", "max"):
        raise ValueError(f"`objective_sense` was expected as 'min' or 'max', but it was received as {objective_sense!r}")
    center_init = torch.as_tensor(center_init)
    if not center_init.is_floating_point():
        center_init = center_init.to(torch.get_default_dtype())
    if center_init.ndim < 1 or center_init.shape[-1] == 0:
        raise ValueError(f"`center_init` was expected with shape (..., D), D >= 1; got {tuple(center_init.shape)}")
    d = center_init.shape[-1]
    stdev = vector_like_center(stdev_init, "stdev_init", center_init)
    batch = tuple(torch.broadcast_shapes(center_init.shape[:-1], stdev.shape[:-1]))
    center = center_init.expand(batch + (d,)).contiguous().clone()
    popsize = default_popsize(d) if popsize is None else int(popsize)
    if popsize < 2:
        raise ValueError(f"`popsize` must be at least 2, got {popsize}")
    default_lr = 0.2 * (3 + math.log(d)) / math.sqrt(d)
    lr_sigma = default_lr if stdev_learning_rate is None else float(stdev_learning_rate) * (default_lr if scale_learning_rate else 1.0)
    lr_mu = 1.0 if center_learning_rate is None else float(center_learning_rate)
    optimizer_state = None
    if optimizer is not None:
        init, _, _ = get_functional_optimizer(optimizer)
        optimizer_state = init(center_init=center, center_learning_rate=lr_mu, **(optimizer_config or {}))
    bound = lambda x, name: None if x is None else vector_like_center(x, name, center_init)  # noqa: E731
    return SNESState(center=center, stdev=stdev.expand(batch + (d,)).contiguous().clone(), optimizer=optimizer, optimizer_state=optimizer_state,
                     popsize=popsize, center_learning_rate=lr_mu, stdev_learning_rate=lr_sigma, stdev_min=bound(stdev_min, "stdev_min"),
                     stdev_max=bound(stdev_max, "stdev_max"), stdev_max_change=bound(stdev_max_change, "stdev_max_change"),
                     ranking_method=check_ranking_method(ranking_method), maximize=(objective_sense == "max"))


def snes_ask(state: SNESState) -> torch.Tensor:
    """A population per item, (..., popsize, D): row i of item b is mu_b + sigma_b * z_i, z_i ~ N(0, I) (on the kernels, the
    batched Philox sampler, item b on stream b)."""
    return sample_separable(state.center, state.stdev, state.popsize, False)


def snes_ask_and_evaluate(state: SNESState, *, objective: Callable, lazy: bool = False) -> tuple:
    """`snes_ask` and the fitnesses of the population: (values (..., popsize, D), evals (..., popsize)).  With the state on the
    kernels and an objective with a fused kernel, all items are sampled and evaluated in one launch; with `lazy=True` the
    population is not stored either, and `values` is a `LazyPopulation` that `snes_tell` takes in place of the tensor (its
    gradient rows are rebuilt from their Philox counters, bit-identical to the stored population's).  Otherwise this is
    `snes_ask` followed by `objective(values)`, and `lazy=True` raises ValueError."""
    return ask_and_evaluate(lambda: snes_ask(state), state.center, state.stdev, state.popsize, False, objective, lazy)


def _bounds(state: SNESState, batch: tuple) -> tuple:
    return tuple(None if t is None else flat_items(t, batch, 1).contiguous() for t in (state.stdev_min, state.stdev_max, state.stdev_max_change))


def snes_tell(state: SNESState, values: Union[torch.Tensor, LazyPopulation], evals: torch.Tensor) -> SNESState:
    """The next state, given the population `values` (..., popsize, D) and its fitnesses `evals` (..., popsize).  `values` may be
    the LazyPopulation of `snes_ask_and_evaluate(..., lazy=True)` on this very state.  The state passed in is left unchanged."""
    mu, sigma = state.center, state.stdev
    batch, d, n = tuple(mu.shape[:-1]), mu.shape[-1], state.popsize
    lazy = isinstance(values, LazyPopulation)
    if lazy:
        values.check_drawn_from(mu, sigma, False)
    else:
        values = torch.as_tensor(values, dtype=mu.dtype, device=mu.device)
    evals = torch.as_tensor(evals, dtype=mu.dtype, device=mu.device)
    if tuple(values.shape) != batch + (n, d):
        raise ValueError(f"`values` was expected with shape {batch + (n, d)}, got {tuple(values.shape)}")
    if tuple(evals.shape) != batch + (n,):
        raise ValueError(f"`evals` was expected with shape {batch + (n,)}, got {tuple(evals.shape)}")
    B = math.prod(batch)
    mus, sigmas, fs = mu.reshape(B, d), sigma.reshape(B, d), evals.reshape(B, n)
    lbs, ubs, mcs = _bounds(state, batch)
    if lazy or on_kernels(mus, sigmas, values, fs):
        w = ops.rank_batched(fs.contiguous(), state.ranking_method, state.maximize)
        if state.ranking_method != "nes":
            ops.weights_adjust_batched_(w, 2)  # w / sum |w|
        if lazy:
            gmu, gsig = ops.grad_batched_regen(ops.GRAD_EXP, w, mus, sigmas, 1.0, 1.0, seed=values.seed)
        else:
            gmu, gsig = ops.grad_batched(ops.GRAD_EXP, values.reshape(B, n, d), w, mus, sigmas, 1.0, 1.0)
        new_sigma = sigmas.clone()
        ops.sigma_update_batched_(new_sigma, gsig, [state.stdev_learning_rate] * B, True, lb=lbs, ub=ubs, max_change=mcs)
        new_mu = None
        if state.optimizer is None:
            new_mu = mus.clone()
            ops.axpy_(new_mu.view(-1), gmu.view(-1), state.center_learning_rate)
    else:
        x = values.reshape(B, n, d)
        w = rank_rows(fs, state.ranking_method, state.maximize)
        if state.ranking_method != "nes":
            w = w / w.abs().sum(-1, keepdim=True)
        eps = x - mus[:, None, :]
        gmu = torch.einsum("bn,bnd->bd", w, eps)
        gsig = torch.einsum("bn,bnd->bd", w, (eps / sigmas[:, None, :]) ** 2 - 1)
        new_sigma = modify_tensor(sigmas, sigmas * torch.exp(0.5 * (state.stdev_learning_rate * gsig)), lb=lbs, ub=ubs, max_change=mcs)
        new_mu = None if state.optimizer is not None else mus + state.center_learning_rate * gmu
    new = dict(stdev=new_sigma.view(batch + (d,)))
    if state.optimizer is None:
        new["center"] = new_mu.view(batch + (d,))
    else:
        _, ask, tell = get_functional_optimizer(state.optimizer)
        new["optimizer_state"] = tell(state.optimizer_state, follow_grad=gmu.view(batch + (d,)))
        new["center"] = ask(new["optimizer_state"])
    return state._replace(**new)
