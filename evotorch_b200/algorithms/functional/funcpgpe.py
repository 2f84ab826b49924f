"""Functional PGPE: `pgpe(...) -> PGPEState`, `pgpe_ask(state, popsize=...)`, `pgpe_tell(state, values, evals)`
(reference: algorithms/functional/funcpgpe.py:54-384).

The arithmetic is the one of the object-oriented PGPE (SURVEY 8 rows a2, a4-a9): sampling K1, ranking K3, the utility-weighted
reductions K4 and the ClipUp / Adam / SGD + clamped-sigma updates K5 -- here driven per batch item with explicit state.
"""

from __future__ import annotations

import os

from typing import Callable, NamedTuple, Optional, Union

import torch

from ... import ops
from ...distributions import SeparableGaussian, SymmetricSeparableGaussian
from ...tools import modify_tensor
from .fused import LazyPopulation, ask_and_evaluate
from .misc import (batch_shape_of, draw_philox_seed, expand_to, flat_items, get_functional_optimizer, get_stdev_init, host_scalar, on_kernels,
                   scalar_items, vector_like_center)


class PGPEState(NamedTuple):
    optimizer: Union[str, tuple]
    optimizer_state: tuple
    stdev: torch.Tensor
    stdev_learning_rate: torch.Tensor
    stdev_min: torch.Tensor
    stdev_max: torch.Tensor
    stdev_max_change: torch.Tensor
    ranking_method: str
    maximize: bool
    symmetric: bool


def pgpe(*, center_init, center_learning_rate, stdev_learning_rate, objective_sense: str, ranking_method: str = "centered",
         optimizer: Union[str, tuple] = "clipup", optimizer_config: Optional[dict] = None, stdev_init=None, radius_init=None, stdev_min=None,
         stdev_max=None, stdev_max_change=0.2, symmetric: bool = True) -> PGPEState:
    """Initial PGPE state (defaults as funcpgpe.py:69-85: symmetric sampling, ClipUp, centered ranking, sigma moves <= 20 %)."""
    center_init = torch.as_tensor(center_init)
    if center_init.ndim < 1:
        raise ValueError(f"The center of the search distribution for the functional PGPE was expected as a tensor with at least 1 dimension."
                         f" However, the encountered `center` is {center_init}, of shape {center_init.shape}.")
    if center_init.shape[-1] == 0:
        raise ValueError("Solution length cannot be 0")
    if objective_sense not in ("min", "max"):
        raise ValueError(f"`objective_sense` was expected as 'min' or 'max', but it was received as {objective_sense!r}")
    dtype = center_init.dtype
    init, _, _ = get_functional_optimizer(optimizer)
    optimizer_state = init(center_init=center_init, center_learning_rate=host_scalar(center_learning_rate, dtype), **(optimizer_config or {}))
    return PGPEState(
        optimizer=optimizer,
        optimizer_state=optimizer_state,
        stdev=get_stdev_init(center_init=center_init, stdev_init=stdev_init, radius_init=radius_init),
        stdev_learning_rate=host_scalar(stdev_learning_rate, dtype),
        stdev_min=vector_like_center(0.0 if stdev_min is None else stdev_min, "stdev_min", center_init),
        stdev_max=vector_like_center(float("inf") if stdev_max is None else stdev_max, "stdev_max", center_init),
        stdev_max_change=vector_like_center(float("inf") if stdev_max_change is None else stdev_max_change, "stdev_max_change", center_init),
        ranking_method=str(ranking_method),
        maximize=(objective_sense == "max"),
        symmetric=bool(symmetric),
    )


def _distribution(symmetric: bool, mu: torch.Tensor, sigma: torch.Tensor):
    if symmetric:
        return SymmetricSeparableGaussian({"mu": mu, "sigma": sigma, "divide_mu_grad_by": "num_directions",
                                           "divide_sigma_grad_by": "num_directions"})
    return SeparableGaussian({"mu": mu, "sigma": sigma, "divide_mu_grad_by": "num_solutions", "divide_sigma_grad_by": "num_solutions"})


def sample_separable(center: torch.Tensor, stdev: torch.Tensor, popsize: int, symmetric: bool) -> torch.Tensor:
    """(..., popsize, D) samples of N(center, diag(stdev^2)), antithetic pairs in rows (2k, 2k+1) when `symmetric`."""
    batch = batch_shape_of((center, 1), (stdev, 1))
    d = center.shape[-1]
    popsize = int(popsize)
    if symmetric and popsize % 2 != 0:
        raise ValueError(f"Symmetric sampling cannot be done if the number of solutions is odd: {popsize}")
    out = torch.empty(tuple(batch) + (popsize, d), dtype=center.dtype, device=center.device)
    mus, sigmas, outs = flat_items(center, batch, 1), flat_items(stdev, batch, 1), out.view(-1, popsize, d)
    if on_kernels(center, stdev):
        # K1, ONE launch for all batch items (grid y = item); the batch index is the Philox stream, so the items are independent
        # draws of one key
        ops.sample_batched(outs, mus if center.ndim > 1 else center, sigmas if stdev.ndim > 1 else stdev, symmetric=symmetric,
                           seed=draw_philox_seed())
    else:
        for b in range(outs.shape[0]):
            _distribution(symmetric, mus[b], sigmas[b]).sample(out=outs[b])
    return out


def pgpe_ask(state: PGPEState, *, popsize: int) -> torch.Tensor:
    """A population of `popsize` solutions: a tensor of shape (..., popsize, solution_length)."""
    _, ask, _ = get_functional_optimizer(state.optimizer)
    return sample_separable(ask(state.optimizer_state), state.stdev, popsize, state.symmetric)


def pgpe_ask_and_evaluate(state: PGPEState, *, popsize: int, objective: Callable, lazy: bool = False) -> tuple:
    """`pgpe_ask` and the fitnesses of the population: (values (..., popsize, L), evals (..., popsize)).

    With the centre and stdev on the kernels (float32 CUDA) and an objective with a fused kernel (`evok_objective_id`: the
    objectives of evotorch_b200.objectives and every FusedObjective), the populations of all batch items are sampled and evaluated
    in one launch: the population is written once and not read back for the evaluation, and under the same torch.manual_seed it
    is the population `pgpe_ask` would return.  `lazy=True` does not store it either: `values` is then a `LazyPopulation`, which
    `pgpe_tell` takes in place of the tensor and whose gradient rows are rebuilt from their Philox counters, bit-identical to the
    stored population's.  (A tell whose batch is larger than the population's -- batched hyper-parameters over an unbatched
    centre and stdev -- regenerates the population for that tell: it broadcasts one drawn item to several.)  Otherwise this is `pgpe_ask` followed by `objective(values)`, and `lazy=True` raises ValueError."""
    _, ask, _ = get_functional_optimizer(state.optimizer)
    return ask_and_evaluate(lambda: pgpe_ask(state, popsize=popsize), ask(state.optimizer_state), state.stdev, popsize, state.symmetric, objective,
                            lazy)


def pgpe_tell(state: PGPEState, values: Union[torch.Tensor, LazyPopulation], evals: torch.Tensor) -> PGPEState:
    """The next state, given the population `values` (..., N, L) and its fitnesses `evals` (..., N).  `values` may be the
    LazyPopulation of `pgpe_ask_and_evaluate(..., lazy=True)` on this very state."""
    _, ask, tell = get_functional_optimizer(state.optimizer)
    center = ask(state.optimizer_state)
    lazy = isinstance(values, LazyPopulation)
    if lazy:
        values.check_drawn_from(center, state.stdev, state.symmetric)
    else:
        values = torch.as_tensor(values, dtype=center.dtype, device=center.device)
    evals = torch.as_tensor(evals, dtype=center.dtype, device=center.device)
    lr_sigma = state.stdev_learning_rate
    batch = batch_shape_of((center, 1), (state.stdev, 1), (values, 2), (evals, 1), (lr_sigma, 0), (state.stdev_min, 1), (state.stdev_max, 1),
                           (state.stdev_max_change, 1))
    if lazy and tuple(batch) != tuple(values.shape[:-2]):
        # batched hyper-parameters or fitnesses over fewer population items: the tell broadcasts a drawn item to several of its
        # items, which the rebuild (item b on stream b) cannot; the population is regenerated bit for bit for this tell instead
        values, lazy = values.materialize(), False
    d = center.shape[-1]
    mus, sigmas = flat_items(center, batch, 1), flat_items(state.stdev, batch, 1)
    xs = None if lazy else flat_items(values, batch, 2)
    fs = flat_items(evals, batch, 1)
    lbs, ubs, mcs = (flat_items(t, batch, 1) for t in (state.stdev_min, state.stdev_max, state.stdev_max_change))
    sense = "max" if state.maximize else "min"
    n_items = mus.shape[0]
    grad_mu = torch.empty(n_items, d, dtype=center.dtype, device=center.device)
    new_stdev = expand_to(state.stdev, batch, 1).contiguous().clone()
    new_sigmas = new_stdev.view(-1, d)
    kernels = lazy or on_kernels(center, values)
    if lazy or (kernels and os.environ.get("EVOTORCH_B200_FUNCTIONAL_LOOP", "0") != "1"):  # (=1: the per-item launch chains, for comparison)
        # one launch per stage for ALL batch items (grid y / z = item): K3 ranking, K4 weighted reductions, K5 sigma update
        n = fs.shape[1]
        w = ops.rank_batched(fs, state.ranking_method, state.maximize)
        if state.ranking_method not in ("centered", "normalized"):  # distributions.py:562-563 / :722-723: w - mean(w)
            ops.weights_adjust_batched_(w, 1)
        scale = 1.0 / (n // 2) if state.symmetric else 1.0 / n  # divide by num_directions / num_solutions (funcpgpe.py defaults)
        form = ops.GRAD_SYMMETRIC if state.symmetric else ops.GRAD_SEPARABLE
        mu_items, sigma_items = mus if center.ndim > 1 else center, sigmas if state.stdev.ndim > 1 else state.stdev
        if lazy:  # the rows with a non-zero weight, rebuilt from their Philox counters: the bits of the stored population's gradient
            gmu, gsig = ops.grad_batched_regen(form, w, mu_items, sigma_items, scale, scale, seed=values.seed)
        else:
            gmu, gsig = ops.grad_batched(form, xs, w, mu_items, sigma_items, scale, scale)
        ops.sigma_update_batched_(new_sigmas, gsig, scalar_items(lr_sigma, batch), False, lb=lbs.contiguous(), ub=ubs.contiguous(),
                                  max_change=mcs.contiguous())
        new_optimizer_state = tell(state.optimizer_state, follow_grad=gmu.view(tuple(batch) + (d,)))
        return state._replace(optimizer_state=new_optimizer_state, stdev=new_stdev)
    for b, lr_b in enumerate(scalar_items(lr_sigma, batch)):
        dist = _distribution(state.symmetric, mus[b].contiguous(), sigmas[b].contiguous())
        grads = dist.compute_gradients(xs[b], fs[b], objective_sense=sense, ranking_method=state.ranking_method)  # K3 + K4
        grad_mu[b] = grads["mu"]
        if kernels:  # K5: sigma + lr * grad, clamped to [lb, ub] and to |change| <= max_change * sigma, in one launch
            ops.sigma_update_(new_sigmas[b], grads["sigma"].contiguous(), lr_b, False, lb=lbs[b].contiguous(), ub=ubs[b].contiguous(),
                              max_change=mcs[b].contiguous())
        else:
            new_sigmas[b] = modify_tensor(sigmas[b], sigmas[b] + lr_b * grads["sigma"], lb=lbs[b], ub=ubs[b], max_change=mcs[b])
    new_optimizer_state = tell(state.optimizer_state, follow_grad=grad_mu.view(tuple(batch) + (d,)))
    return state._replace(optimizer_state=new_optimizer_state, stdev=new_stdev)
