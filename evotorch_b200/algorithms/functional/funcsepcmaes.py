"""Functional separable CMA-ES: `sepcmaes(...) -> SepCMAESState`, `sepcmaes_ask(state)`, `sepcmaes_ask_and_evaluate(state, ...)`,
`sepcmaes_tell(state, values, evals)`.

Separable CMA-ES (diagonal covariance), the algorithm of `CMAES(..., separable=True)` (same defaults, hyper-parameters and update
order), with explicit state and extra leftmost batch dimensions: every batch item is an independent search with its own centre,
step size, diagonal covariance and evolution paths; the population size, weights and learning rates are shared.  It scales to
solution lengths where the full-covariance `cmaes` cannot hold its B x D x D matrices.

On CUDA float32 a generation of ALL items is one launch per stage, with s = sigma * A the per-column stdev:
    ask (+ evaluate): x = fmaf(s, z, m), z ~ N(0, I) (batched Philox sampler, item b on stream b, the objective fused in)
    tell: rank-to-weights  ->  the moments sum a_i z_i, sum b_i z_i^2, sum b_i over the steps recovered from the rows,
          z = (x - m) / s (a row pass for q_i = ||z_i||^2, then the column pass)  ->  m, p_sigma, sigma, p_c, C, the stdev
          bounds, A and s (one CTA per item).
With `lazy=True` the population is never stored: the tell rebuilds the rows it needs from their Philox counters, as the sampler
stored them, and its result is bit-identical to telling the stored population.  Nothing is read back to the host: the
generation counter that drives h_sig and the decomposition schedule is a Python int in the state.  Anywhere else the same
algorithm runs as batched torch ops.

`sepcmaes_tell` takes any `values` of the asked shape, so repaired or injected solutions are legal: the steps are recovered from
the values, not remembered from the ask.
"""

from __future__ import annotations

import math
from typing import Callable, NamedTuple, Optional, Union

import torch

from ... import ops
from ...objectives import is_transformed
from ..cmaes import CMAESHyperparameters, cmaes_hyperparameters
from .funccmaes import _assigned_weights, _col, _consts, _h_sig, _host_float, _tier_items
from .fused import LazyPopulation, ask_and_evaluate
from .misc import draw_philox_seed, on_kernels


class SepCMAESState(NamedTuple):
    center: torch.Tensor  # (..., D)
    sigma: torch.Tensor  # (...)
    C: torch.Tensor  # (..., D), the diagonal of the covariance
    A: torch.Tensor  # (..., D), its square root as of the last decomposition
    s: torch.Tensor  # (..., D), sigma * A: the per-column stdev the population is drawn with
    p_sigma: torch.Tensor  # (..., D)
    p_c: torch.Tensor  # (..., D)
    generation: int
    hyperparameters: CMAESHyperparameters  # shared by every item: popsize, weights and learning rates
    maximize: bool
    active: bool
    csa_squared: bool
    stdev_min: Optional[float]
    stdev_max: Optional[float]

    @property
    def popsize(self) -> int:
        return self.hyperparameters.popsize

    @property
    def weights(self) -> torch.Tensor:
        return self.hyperparameters.weights


def sepcmaes(*, center_init, stdev_init, objective_sense: str, popsize: Optional[int] = None, c_m: float = 1.0, c_sigma_ratio: float = 1.0,
             damp_sigma_ratio: float = 1.0, c_c_ratio: float = 1.0, c_1_ratio: float = 1.0, c_mu_ratio: float = 1.0, active: bool = True,
             csa_squared: bool = False, stdev_min: Optional[float] = None, stdev_max: Optional[float] = None,
             limit_C_decomposition: bool = True) -> SepCMAESState:
    """Initial state.  `center_init` (..., D); `stdev_init` a scalar or a tensor of batch shape; the batch shape of the search is
    their broadcast.  Defaults and derived constants are those of `CMAES(..., separable=True)` with the same arguments."""
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
    ratios = {name: _host_float(v, name) for name, v in (("c_m", c_m), ("c_sigma_ratio", c_sigma_ratio), ("damp_sigma_ratio", damp_sigma_ratio),
                                                          ("c_c_ratio", c_c_ratio), ("c_1_ratio", c_1_ratio), ("c_mu_ratio", c_mu_ratio))}
    hp = cmaes_hyperparameters(d, popsize, dtype=dtype, device=device, active=active, separable=True,
                               limit_C_decomposition=limit_C_decomposition, **ratios)
    sigma = sigma.expand(batch).contiguous().clone()
    ones = torch.ones(batch + (d,), dtype=dtype, device=device)
    return SepCMAESState(
        center=center_init.expand(batch + (d,)).contiguous().clone(),
        sigma=sigma,
        C=ones.clone(),
        A=ones.clone(),
        s=sigma[..., None] * ones,
        p_sigma=torch.zeros(batch + (d,), dtype=dtype, device=device),
        p_c=torch.zeros(batch + (d,), dtype=dtype, device=device),
        generation=0,
        hyperparameters=hp,
        maximize=(objective_sense == "max"),
        active=bool(active),
        csa_squared=bool(csa_squared),
        stdev_min=None if stdev_min is None else _host_float(stdev_min, "stdev_min"),
        stdev_max=None if stdev_max is None else _host_float(stdev_max, "stdev_max"),
    )


def _items(state: SepCMAESState) -> tuple:
    """(batch shape, number of items B, D) of a state."""
    batch, d = tuple(state.center.shape[:-1]), state.center.shape[-1]
    return batch, math.prod(batch), d


def _ask(state: SepCMAESState) -> tuple:
    """(`sepcmaes_ask`'s population, the Philox seed of its draw on the kernels (item b on stream b), None elsewhere)."""
    batch, B, d = _items(state)
    n = state.popsize
    m, s = state.center.reshape(B, d), state.s.reshape(B, d)
    seed = None
    if on_kernels(m, s):
        x = torch.empty(B, n, d, dtype=torch.float32, device=m.device)
        seed = draw_philox_seed()
        ops.sample_batched(x, m, s, symmetric=False, seed=seed)
    else:
        x = m[:, None, :] + s[:, None, :] * torch.randn(B, n, d, dtype=m.dtype, device=m.device)
    return x.view(batch + (n, d)), seed


def sepcmaes_ask(state: SepCMAESState) -> torch.Tensor:
    """A population per item: a tensor of shape (..., popsize, D), row i of item b = m_b + s_b * z_i (on the kernels
    fmaf(s_b, z_i, m_b), one launch of the batched sampler for all items, item b on Philox stream b)."""
    return _ask(state)[0]


def sepcmaes_ask_and_evaluate(state: SepCMAESState, *, objective: Callable, lazy: bool = False) -> tuple:
    """`sepcmaes_ask` and the fitnesses of the population: (values (..., popsize, D), evals (..., popsize)).

    With the state on the kernels (float32 CUDA) and an objective with a fused kernel (`evok_objective_id`: the objectives of
    evotorch_b200.objectives and every FusedObjective), the populations of all items are sampled and evaluated in one launch;
    under the same torch.manual_seed the stored population is the one `sepcmaes_ask` would return.  `lazy=True` does not store it:
    `values` is then a `LazyPopulation`, which `sepcmaes_tell` takes in place of the tensor.  Otherwise this is `sepcmaes_ask`
    followed by `objective(values)`, and `lazy=True` raises ValueError.  An objective whose data has a batch shape must have the
    state's batch shape: a CMA-ES state is not broadcast to more items.  A FusedObjective with a transform has no fused sampler:
    the population is stored and its kernels evaluate it, keyed with the ask's Philox draw (so a noisy one gets the noise the
    batched sampler would give it)."""
    batch, _, _ = _items(state)
    per_item = tuple(getattr(objective, "data_batch_shape", ()))
    if per_item and per_item != batch:
        raise ValueError(f"the data of {objective!r} has batch shape {per_item}, the separable CMA-ES state {batch}: each item of the data "
                         "needs its own search (build the state with that batch shape)")
    if is_transformed(objective) and not lazy:
        values, seed = _ask(state)
        return values, (objective(values) if seed is None else objective.evaluate_batched(values, seed=seed))
    return ask_and_evaluate(lambda: sepcmaes_ask(state), state.center, state.s, state.popsize, False, objective, lazy)


def sepcmaes_tell(state: SepCMAESState, values: Union[torch.Tensor, LazyPopulation], evals: torch.Tensor) -> SepCMAESState:
    """The next state, given a population `values` (..., popsize, D) -- or the LazyPopulation that `sepcmaes_ask_and_evaluate`
    returned for this very state -- and its fitnesses `evals` (..., popsize).  The state passed in is left unchanged."""
    return _tell(state, values, evals, state.generation)[0]


def _tell(state: SepCMAESState, values: Union[torch.Tensor, LazyPopulation], evals: torch.Tensor, steps, tiers=None) -> tuple:
    """(`sepcmaes_tell`'s next state, the generation counters after it).  `steps` drives h_sig and the decomposition schedule: the
    int `state.generation`, or a (B,) int64 tensor of per-item counters.  `tiers`: as in funccmaes._tell (a padded population:
    item b is told its first ladder.popsizes[tier[b]] rows with the constants and decomposition schedule of its tier)."""
    batch, B, d = _items(state)
    n = state.popsize
    m0 = state.center
    lazy = isinstance(values, LazyPopulation)
    if lazy:
        values.check_drawn_from(state.center, state.s, False)
    else:
        values = torch.as_tensor(values, dtype=m0.dtype, device=m0.device)
    evals = torch.as_tensor(evals, dtype=m0.dtype, device=m0.device)
    if tuple(values.shape) != batch + (n, d):
        raise ValueError(f"`values` was expected with shape {batch + (n, d)}, got {tuple(values.shape)}")
    if tuple(evals.shape) != batch + (n,):
        raise ValueError(f"`evals` was expected with shape {batch + (n,)}, got {tuple(evals.shape)}")
    f = evals.reshape(B, n)
    per_item = isinstance(steps, torch.Tensor)
    if lazy or on_kernels(m0, values, f):
        counters = steps.clone() if per_item else steps  # the kernel increments per-item counters in place
        new = _tell_kernels(state, B, n, d, values, f, counters, tiers)
        steps_next = counters if per_item else steps + 1
    else:
        new = _tell_torch(state, B, n, d, values.reshape(B, n, d), f, steps, tiers)
        steps_next = steps + 1
    m, sigma, C, A, s, p_sigma, p_c = new
    vec = batch + (d,)
    new_state = state._replace(center=m.view(vec), sigma=sigma.view(batch), C=C.view(vec), A=A.view(vec), s=s.view(vec), p_sigma=p_sigma.view(vec),
                               p_c=p_c.view(vec), generation=state.generation + 1)
    return new_state, steps_next


def _tell_kernels(state, B, n, d, values, f, steps, tiers=None) -> tuple:
    """Rank table, moments (row pass + column pass) and update, one launch each for all items; every output is a new tensor.
    `steps`: the shared int counter, or the per-item int64 counters, which the update increments.  `tiers`: as in `_tell`; the
    moments never read (or rebuild) a pad row, whose weight is 0."""
    hp = state.hyperparameters
    lazy = isinstance(values, LazyPopulation)
    m, s = state.center.reshape(B, d).contiguous(), state.s.reshape(B, d).contiguous()
    if tiers is None:
        aw = ops.rank_table_batched(f, state.maximize, hp.weights)
        consts, freq, tier = _consts(hp), hp.decompose_C_freq, None
    else:
        ladder, tier = tiers
        aw = ops.rank_table_batched(f, state.maximize, ladder.weights, tier=tier, counts=ladder.counts)
        consts, freq = ladder.consts, ladder.decompose_C_freq
    X = None if lazy else values.reshape(B, n, d).contiguous()
    local, S2, wsum = ops.sepcma_moments_batched(X, m, s, aw, state.active, seed=values.seed if lazy else 0)
    out = [t.reshape(B, d).clone() for t in (state.center, state.C, state.A, state.s, state.p_sigma, state.p_c)]
    m_new, C, A, s_new, p_sigma, p_c = out
    sigma = state.sigma.reshape(B).clone()
    ops.sepcma_update_batched(local, S2, wsum, m_new, p_sigma, p_c, sigma, C, A, s_new, consts, state.csa_squared, steps=steps,
                              decompose_C_freq=freq, stdev_min=state.stdev_min, stdev_max=state.stdev_max, tier=tier)
    return m_new, sigma, C, A, s_new, p_sigma, p_c


def _tell_torch(state, B, n, d, x, f, steps, tiers=None) -> tuple:
    """The same generation as batched torch ops (CMAES's op-by-op generation with separable=True, cmaes.py:454-565), with the
    generation counter `steps` (an int, or per-item counters).  `tiers`: as in `_tell` (the constants become per-item tensors)."""
    hp = state.hyperparameters
    m, sigma, C, A, s = state.center.reshape(B, d), state.sigma.reshape(B), state.C.reshape(B, d), state.A.reshape(B, d), state.s.reshape(B, d)
    if tiers is not None:  # pad rows at the centre: their z is exactly 0, whatever they held
        hp, weights, real = _tier_items(tiers, n)
        x = torch.where(real[:, :, None], x, m[:, None, :])
    z = (x - m[:, None, :]) / s[:, None, :]
    zz = z * z
    aw = _assigned_weights(f, state.maximize, hp.weights) if tiers is None else _assigned_weights(f, state.maximize, weights, real)
    a = torch.clamp_min(aw, 0.0)
    b = torch.where(aw < 0, d * aw / zz.sum(-1), aw) if state.active else aw
    local = torch.einsum("bn,bnd->bd", a, z)
    S2 = torch.einsum("bn,bnd->bd", b, zz)
    wsum = b.sum(-1)
    shaped = A * local
    m = m + _col(hp.c_m) * sigma[:, None] * shaped
    p_sigma = _col(1 - hp.c_sigma) * state.p_sigma.reshape(B, d) + _col(hp.variance_discount_sigma) * local
    pnorm = torch.linalg.vector_norm(p_sigma, dim=-1)
    if state.csa_squared:
        expo = (pnorm.pow(2.0) / d - 1) / 2
    else:
        expo = pnorm / hp.unbiased_expectation - 1
    sigma = sigma * torch.exp((hp.c_sigma / hp.damp_sigma) * expo)
    h_sig = _h_sig(hp, pnorm, d, steps)
    p_c = _col(1 - hp.c_c) * state.p_c.reshape(B, d) + (h_sig * hp.variance_discount_c)[:, None] * shaped
    c1a = hp.c_1 * (1 - (1 - h_sig**2) * hp.c_c * (2 - hp.c_c))
    C = C + c1a[:, None] * (p_c.pow(2.0) - C) + _col(hp.c_mu) * (A.pow(2.0) * S2 - wsum[:, None] * C)
    if state.stdev_min is not None or state.stdev_max is not None:  # CMAES._limit_stdev, with the new sigma
        stdevs = torch.clamp(sigma[:, None] * torch.sqrt(C), min=state.stdev_min, max=state.stdev_max)
        C = (stdevs / sigma[:, None]).pow(2.0)
    if isinstance(steps, torch.Tensor):
        A = torch.where(((steps + 1) % hp.decompose_C_freq == 0)[:, None], C.pow(0.5), A)
    elif (steps + 1) % hp.decompose_C_freq == 0:
        A = C.pow(0.5)
    return m, sigma, C, A, sigma[:, None] * A, p_sigma, p_c
