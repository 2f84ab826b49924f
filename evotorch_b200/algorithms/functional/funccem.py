"""Functional cross-entropy method: `cem(...) -> CEMState`, `cem_ask`, `cem_tell`
(reference: algorithms/functional/funccem.py:24-289; Rubinstein 1999, as in Duan et al. 2016).

tell: elites = the best floor(N * parenthood_ratio) solutions; center <- mean(elites); stdev <- std(elites, unbiased),
then clamped against the old stdev (SURVEY 8 rows a6 + a8; kernels K3, K4 in its raw-moments form, K5).
"""

from __future__ import annotations

import os

from typing import Callable, NamedTuple, Union

import torch

from ... import ops
from ...distributions import SeparableGaussian
from ...tools import modify_tensor
from .funcpgpe import sample_separable
from .fused import LazyPopulation, ask_and_evaluate
from .misc import batch_shape_of, expand_to, flat_items, get_stdev_init, on_kernels, vector_like_center


class CEMState(NamedTuple):
    center: torch.Tensor
    stdev: torch.Tensor
    stdev_min: torch.Tensor
    stdev_max: torch.Tensor
    stdev_max_change: torch.Tensor
    parenthood_ratio: float
    maximize: bool


def cem(*, center_init, parenthood_ratio: float, objective_sense: str, stdev_init=None, radius_init=None, stdev_min=None, stdev_max=None,
        stdev_max_change=None) -> CEMState:
    center_init = torch.as_tensor(center_init)
    if center_init.ndim < 1:
        raise ValueError(f"The center of the search distribution for the functional CEM was expected as a tensor with at least 1 dimension."
                         f" However, the encountered `center_init` is {center_init}, of shape {center_init.shape}.")
    if center_init.shape[-1] == 0:
        raise ValueError("Solution length cannot be 0")
    if objective_sense not in ("min", "max"):
        raise ValueError(f"`objective_sense` was expected as 'min' or 'max', but it was received as {objective_sense!r}")
    return CEMState(
        center=center_init,
        stdev=get_stdev_init(center_init=center_init, stdev_init=stdev_init, radius_init=radius_init),
        stdev_min=vector_like_center(0.0 if stdev_min is None else stdev_min, "stdev_min", center_init),
        stdev_max=vector_like_center(float("inf") if stdev_max is None else stdev_max, "stdev_max", center_init),
        stdev_max_change=vector_like_center(float("inf") if stdev_max_change is None else stdev_max_change, "stdev_max_change", center_init),
        parenthood_ratio=float(parenthood_ratio),
        maximize=(objective_sense == "max"),
    )


def cem_ask(state: CEMState, *, popsize: int) -> torch.Tensor:
    return sample_separable(state.center, state.stdev, popsize, False)


def cem_ask_and_evaluate(state: CEMState, *, popsize: int, objective: Callable, lazy: bool = False) -> tuple:
    """`cem_ask` and the fitnesses of the population, fused into one launch where the kernels and the objective allow it; see
    `pgpe_ask_and_evaluate`.  With `lazy=True` the tell rebuilds only the elites."""
    return ask_and_evaluate(lambda: cem_ask(state, popsize=popsize), state.center, state.stdev, popsize, False, objective, lazy)


def cem_tell(state: CEMState, values: Union[torch.Tensor, LazyPopulation], evals: torch.Tensor) -> CEMState:
    center = state.center
    lazy = isinstance(values, LazyPopulation)
    if lazy:
        values.check_drawn_from(center, state.stdev, False)
    else:
        values = torch.as_tensor(values, dtype=center.dtype, device=center.device)
    evals = torch.as_tensor(evals, dtype=center.dtype, device=center.device)
    batch = batch_shape_of((center, 1), (state.stdev, 1), (values, 2), (evals, 1), (state.stdev_min, 1), (state.stdev_max, 1),
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
    new_center = expand_to(center, batch, 1).contiguous().clone()
    new_stdev = expand_to(state.stdev, batch, 1).contiguous().clone()
    new_mus, new_sigmas = new_center.view(-1, d), new_stdev.view(-1, d)
    kernels = lazy or on_kernels(center, values)
    sense = "max" if state.maximize else "min"
    if lazy or (kernels and os.environ.get("EVOTORCH_B200_FUNCTIONAL_LOOP", "0") != "1"):  # (=1: the per-item launch chains, for comparison)
        # one launch per stage for ALL batch items: raw utilities, elite flags, elite moments, mean / std of the elites, clamped update
        import math

        n = fs.shape[1]
        num_elites = math.floor(n * state.parenthood_ratio)
        w = ops.rank_batched(fs, "raw", state.maximize)
        mask = ops.elite_mask_batched(w, num_elites)
        mu_items, sigma_items = mus if center.ndim > 1 else center, sigmas if state.stdev.ndim > 1 else state.stdev
        if lazy:  # only the elites (non-zero mask) are rebuilt from their Philox counters
            s1, s2 = ops.grad_batched_regen(ops.GRAD_MOMENTS, mask, mu_items, sigma_items, 1.0, 1.0, seed=values.seed)
        else:
            s1, s2 = ops.grad_batched(ops.GRAD_MOMENTS, xs, mask, mu_items, sigma_items, 1.0, 1.0)
        B = s1.shape[0]
        gmu, gsig = ops.cem_finalize(s1.view(-1), s2.view(-1), new_sigmas.reshape(-1), num_elites)
        ops.axpy_(new_mus.view(-1), gmu, 1.0)
        ops.sigma_update_batched_(new_sigmas, gsig.view(B, d), [1.0] * B, False, lb=lbs.contiguous(), ub=ubs.contiguous(), max_change=mcs.contiguous())
        return state._replace(center=new_center, stdev=new_stdev)
    for b in range(mus.shape[0]):
        dist = SeparableGaussian({"mu": mus[b].contiguous(), "sigma": sigmas[b].contiguous(), "parenthood_ratio": state.parenthood_ratio})
        grads = dist.compute_gradients(xs[b], fs[b], objective_sense=sense)  # mean(elites) - mu, std(elites) - sigma
        if kernels:
            ops.axpy_(new_mus[b], grads["mu"].contiguous(), 1.0)
            ops.sigma_update_(new_sigmas[b], grads["sigma"].contiguous(), 1.0, False, lb=lbs[b].contiguous(), ub=ubs[b].contiguous(),
                              max_change=mcs[b].contiguous())
        else:
            new_mus[b] = mus[b] + grads["mu"]
            new_sigmas[b] = modify_tensor(sigmas[b], sigmas[b] + grads["sigma"], lb=lbs[b], ub=ubs[b], max_change=mcs[b])
    return state._replace(center=new_center, stdev=new_stdev)
