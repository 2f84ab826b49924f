"""Functional CMA-ES: `cmaes(...) -> CMAESState`, `cmaes_ask(state)`, `cmaes_tell(state, values, evals)`.

Full-covariance CMA-ES with active weights, the algorithm of `algorithms.cmaes.CMAES` (same defaults, hyper-parameters and update
order), with explicit state and extra leftmost batch dimensions: every batch item is an independent search with its own centre,
step size, covariance, Cholesky factor and evolution paths; the population size, weights and learning rates are shared.

On CUDA float32 a generation of ALL items is one launch per stage:
    ask : z ~ N(0, I) (batched Philox sampler, item b on stream b)  ->  x = m_b + sigma_b z A_b^T (batched 3xTF32 GEMM, affine epilogue)
    tell: y = (x - m) / sigma, z = A^-1 y (batched triangular solve)  ->  rank-to-weights  ->  row weights  ->  sum w z, sum w y
          (batched weighted row sums)  ->  m, p_sigma, sigma, h_sig, p_c (one CTA per item)  ->  weighted SYRK with the covariance
          update in its epilogue  ->  stdev bounds on the diagonal  ->  Cholesky of the (B, D, D) stack on the decomposition schedule.
Nothing is read back to the host: the generation counter that drives h_sig and the schedule is a Python int in the state.
Anywhere else the same algorithm runs as batched torch ops.

`cmaes_ask_and_evaluate(state, objective=...)` asks and evaluates: with an objective that has a fused kernel, the fitnesses of all
items come from one launch of the batched evaluation kernel, keyed with the ask's Philox draw (per-item data, noise of the draw).

`cmaes_tell` takes any `values` of the asked shape, so repaired or injected solutions are legal (as in pycma's `tell`): the
steps z are recovered from the values, not remembered from the ask.
"""

from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Callable, NamedTuple, Optional

import torch

from ... import ops
from ..cmaes import CMAESHyperparameters, cmaes_hyperparameters
from .fused import LazyPopulation, ask_and_evaluate_keyed
from .misc import draw_philox_seed, on_kernels


class CMAESState(NamedTuple):
    center: torch.Tensor  # (..., D)
    sigma: torch.Tensor  # (...)
    C: torch.Tensor  # (..., D, D)
    A: torch.Tensor  # (..., D, D), lower Cholesky factor of C as of the last decomposition
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


def _host_float(x, name: str) -> float:
    """A hyper-parameter that every item shares, as a Python float (a batch of values is rejected)."""
    if isinstance(x, torch.Tensor):
        if x.numel() != 1:
            raise ValueError(f"`{name}` must be one value shared by every batch item; per-item values are not supported (got shape {tuple(x.shape)})")
        x = x.item()
    return float(x)


def cmaes(*, center_init, stdev_init, objective_sense: str, popsize: Optional[int] = None, c_m: float = 1.0, c_sigma_ratio: float = 1.0,
          damp_sigma_ratio: float = 1.0, c_c_ratio: float = 1.0, c_1_ratio: float = 1.0, c_mu_ratio: float = 1.0, active: bool = True,
          csa_squared: bool = False, stdev_min: Optional[float] = None, stdev_max: Optional[float] = None, limit_C_decomposition: bool = True,
          separable: bool = False) -> CMAESState:
    """Initial state.  `center_init` (..., D); `stdev_init` a scalar or a tensor of batch shape; the batch shape of the search is
    their broadcast.  Defaults and derived constants are those of `CMAES` with the same arguments."""
    if separable:
        raise ValueError("The functional CMA-ES is the full-covariance algorithm; separable CMA-ES is available as CMAES(separable=True)")
    if objective_sense not in ("min", "max"):
        raise ValueError(f"`objective_sense` was expected as 'min' or 'max', but it was received as {objective_sense!r}")
    center_init = torch.as_tensor(center_init)
    if not center_init.is_floating_point():
        center_init = center_init.to(torch.get_default_dtype())
    if center_init.ndim < 1 or center_init.shape[-1] == 0:
        raise ValueError(f"`center_init` was expected with shape (..., D), D >= 1; got {tuple(center_init.shape)}")
    dtype, device, d = center_init.dtype, center_init.device, center_init.shape[-1]
    sigma = torch.as_tensor(stdev_init, dtype=dtype, device=device)
    batch = torch.broadcast_shapes(center_init.shape[:-1], sigma.shape)
    ratios = {name: _host_float(v, name) for name, v in (("c_m", c_m), ("c_sigma_ratio", c_sigma_ratio), ("damp_sigma_ratio", damp_sigma_ratio),
                                                          ("c_c_ratio", c_c_ratio), ("c_1_ratio", c_1_ratio), ("c_mu_ratio", c_mu_ratio))}
    hp = cmaes_hyperparameters(d, popsize, dtype=dtype, device=device, active=active, limit_C_decomposition=limit_C_decomposition, **ratios)
    eye = torch.eye(d, dtype=dtype, device=device).expand(tuple(batch) + (d, d))
    return CMAESState(
        center=center_init.expand(tuple(batch) + (d,)).contiguous().clone(),
        sigma=sigma.expand(batch).contiguous().clone(),
        C=eye.contiguous().clone(),
        A=eye.contiguous().clone(),
        p_sigma=torch.zeros(tuple(batch) + (d,), dtype=dtype, device=device),
        p_c=torch.zeros(tuple(batch) + (d,), dtype=dtype, device=device),
        generation=0,
        hyperparameters=hp,
        maximize=(objective_sense == "max"),
        active=bool(active),
        csa_squared=bool(csa_squared),
        stdev_min=None if stdev_min is None else _host_float(stdev_min, "stdev_min"),
        stdev_max=None if stdev_max is None else _host_float(stdev_max, "stdev_max"),
    )


def _items(state: CMAESState) -> tuple:
    """(batch shape, number of items B, D) of a state."""
    batch, d = tuple(state.center.shape[:-1]), state.center.shape[-1]
    B = math.prod(batch)
    return batch, B, d


def _ask(state: CMAESState) -> tuple:
    """(`cmaes_ask`'s population, the Philox seed of its z on the kernels (item b on stream b), None elsewhere)."""
    batch, B, d = _items(state)
    n = state.popsize
    m, sigma, A = state.center.reshape(B, d), state.sigma.reshape(B), state.A.reshape(B, d, d)
    seed = None
    if on_kernels(m, sigma, A):
        z = torch.empty(B, n, d, dtype=torch.float32, device=m.device)
        zero = torch.zeros(d, dtype=torch.float32, device=m.device)
        seed = draw_philox_seed()
        ops.sample_batched(z, zero, zero + 1.0, symmetric=False, seed=seed)
        x = torch.empty_like(z)
        ops.gemm_nt_batched(z, A.contiguous(), torch.empty_like(z), out2=x, alpha=sigma.contiguous(), bias=m.contiguous())
    else:
        z = torch.randn(B, n, d, dtype=m.dtype, device=m.device)
        x = m[:, None, :] + sigma[:, None, None] * (z @ A.mT)
    return x.view(batch + (n, d)), seed


def cmaes_ask(state: CMAESState) -> torch.Tensor:
    """A population per item: a tensor of shape (..., popsize, D), row i of item b = m_b + sigma_b A_b z_i."""
    return _ask(state)[0]


def cmaes_ask_and_evaluate(state: CMAESState, *, objective: Callable) -> tuple:
    """`cmaes_ask` and the fitnesses of the population: (values (..., popsize, D), evals (..., popsize)).

    With the state on the kernels (float32 CUDA) and an objective with a fused kernel (`evok_objective_id`: the objectives of
    evotorch_b200.objectives and every FusedObjective), the ask runs as `cmaes_ask` does (under the same torch.manual_seed the
    values are bit-identical) and one launch of the batched evaluation kernel evaluates every item, keyed with the Philox draw of
    the z: an objective with noise gives row i of item b the noise the batched sampler would give it, and an objective with
    per-item data gives item b its own data.  Otherwise this is `cmaes_ask` followed by `objective(values)`.  An objective whose
    data has a batch shape must have the state's batch shape.  There is no lazy form: `cmaes_tell` recovers its steps from the
    values."""
    return ask_and_evaluate_keyed(lambda: _ask(state), _items(state)[0], objective, "CMA-ES")


def _limit_stdev(C: torch.Tensor, sigma: torch.Tensor, lo: Optional[float], hi: Optional[float]) -> None:
    """In place on the (B, D, D) stack: diag(C) <- (clamp(sigma sqrt(diag(C)), lo, hi) / sigma)^2 (CMAES._limit_stdev)."""
    if lo is None and hi is None:
        return
    diag = torch.diagonal(C, dim1=-2, dim2=-1)
    stdevs = torch.clamp(sigma[:, None] * torch.sqrt(diag), min=lo, max=hi)
    diag.copy_((stdevs / sigma[:, None]).pow(2.0))


def cmaes_tell(state: CMAESState, values: torch.Tensor, evals: torch.Tensor) -> CMAESState:
    """The next state, given a population `values` (..., popsize, D) and its fitnesses `evals` (..., popsize).  The state passed
    in is left unchanged."""
    return _tell(state, values, evals, state.generation)[0]


def _tell(state: CMAESState, values: torch.Tensor, evals: torch.Tensor, steps, tiers=None) -> tuple:
    """(`cmaes_tell`'s next state, the generation counters after it).  `steps` drives h_sig and the decomposition schedule: the
    int `state.generation`, or a (B,) int64 tensor of per-item counters (then every item is factored and keeps its old A unless
    (steps + 1) % decompose_C_freq == 0 for it).  `tiers` (with per-item counters): None, or (ladder, tier) of a padded
    population (funcrestarts.IPOPLadder, int32 (B,)): item b is told its first ladder.popsizes[tier[b]] rows with the constants of
    its tier, and its pad rows reach nothing."""
    if isinstance(values, LazyPopulation):
        raise ValueError("The functional CMA-ES recovers its steps from the values: a lazy population cannot be told; ask for the values")
    batch, B, d = _items(state)
    n = state.popsize
    m0 = state.center
    values = torch.as_tensor(values, dtype=m0.dtype, device=m0.device)
    evals = torch.as_tensor(evals, dtype=m0.dtype, device=m0.device)
    if tuple(values.shape) != batch + (n, d):
        raise ValueError(f"`values` was expected with shape {batch + (n, d)}, got {tuple(values.shape)}")
    if tuple(evals.shape) != batch + (n,):
        raise ValueError(f"`evals` was expected with shape {batch + (n,)}, got {tuple(evals.shape)}")
    hp = state.hyperparameters
    m, sigma, C, A = m0.reshape(B, d), state.sigma.reshape(B), state.C.reshape(B, d, d), state.A.reshape(B, d, d)
    x, f = values.reshape(B, n, d), evals.reshape(B, n)
    if tiers is not None:  # pad rows at the centre: their y and z are exactly 0, whatever they held
        x = torch.where(_real_rows(tiers, n)[:, :, None], x, m[:, None, :])
    y = (x - m[:, None, :]) / sigma[:, None, None]
    z = torch.linalg.solve_triangular(A.mT, y, upper=True, left=False).contiguous()  # z A^T = y
    per_item = isinstance(steps, torch.Tensor)
    if on_kernels(m, x, f):
        counters = steps.clone() if per_item else steps  # the kernel increments per-item counters in place
        m, p_sigma, p_c, sigma, C_new = _tell_kernels(state, hp, B, n, d, m, sigma, C, y, z, f, counters, tiers)
        steps_next = counters if per_item else steps + 1
    else:
        m, p_sigma, p_c, sigma, C_new = _tell_torch(state, hp, B, n, d, m, sigma, C, y, z, f, steps, tiers)
        steps_next = steps + 1
    _limit_stdev(C_new, sigma, state.stdev_min, state.stdev_max)
    A_new = A
    if per_item:
        A_new, _ = torch.linalg.cholesky_ex(C_new, check_errors=False)
        freq = hp.decompose_C_freq if tiers is None else tiers[0].decompose_C_freq[tiers[1].long()]
        if tiers is not None or hp.decompose_C_freq > 1:
            A_new = torch.where((steps_next % freq == 0)[:, None, None], A_new, A)
    elif (state.generation + 1) % hp.decompose_C_freq == 0:
        A_new, _ = torch.linalg.cholesky_ex(C_new, check_errors=False)
    new = state._replace(center=m.view(batch + (d,)), sigma=sigma.view(batch), C=C_new.view(batch + (d, d)), A=A_new.view(batch + (d, d)),
                         p_sigma=p_sigma.view(batch + (d,)), p_c=p_c.view(batch + (d,)), generation=state.generation + 1)
    return new, steps_next


CONST_NAMES = ("c_m", "c_sigma", "damp_sigma", "c_c", "c_1", "c_mu", "variance_discount_sigma", "variance_discount_c", "unbiased_expectation",
               "weights_sum")  # the order of the 10 constants the update kernels take


def _consts(hp: CMAESHyperparameters) -> tuple:
    return (hp.c_m, hp.c_sigma, hp.damp_sigma, hp.c_c, hp.c_1, hp.c_mu, hp.variance_discount_sigma, hp.variance_discount_c,
            float(hp.unbiased_expectation), hp.weights_sum)


def _real_rows(tiers, n: int) -> torch.Tensor:
    """(B, n) bool: the rows each item of a padded population uses, its first ladder.popsizes[tier] of the n drawn."""
    ladder, tier = tiers
    return torch.arange(n, device=tier.device) < ladder.counts.long()[tier.long()][:, None]


def _tier_items(tiers, n: int) -> tuple:
    """(per-item constants: the names of CONST_NAMES and decompose_C_freq as (B,) tensors, per-item weight rows (B, n), the real
    rows (B, n)) of the items of a padded population at their tiers."""
    ladder, tier = tiers
    t = tier.long()
    c = ladder.consts[t]
    hp = SimpleNamespace(decompose_C_freq=ladder.decompose_C_freq[t], **{name: c[:, k] for k, name in enumerate(CONST_NAMES)})
    return hp, ladder.weights[t], _real_rows(tiers, n)


def _col(v, dims: int = 1):
    """A per-item constant, a (B,) tensor, with `dims` trailing dimensions to meet (B, D) or (B, D, D) operands; a float as is."""
    return v[(slice(None),) + (None,) * dims] if isinstance(v, torch.Tensor) else v


def _tell_kernels(state, hp, B, n, d, m, sigma, C, y, z, f, steps, tiers=None) -> tuple:
    """The stages of CMAES._step_fused for all items at once, one launch each; every output is a new tensor.  `steps`: the shared
    int counter, or the per-item int64 counters, which the vector update increments.  `tiers`: as in `_tell`."""
    dev = m.device
    new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)  # noqa: E731
    aw, w_pos, w_act = new(B, n), new(B, n), new(B, n)
    ladder, tier = tiers if tiers is not None else (None, None)
    tiered = {} if tiers is None else dict(tier=tier, counts=ladder.counts)
    ops.rank_table_batched(f, state.maximize, hp.weights if tiers is None else ladder.weights, out=aw, **tiered)
    ops.cmaes_row_weights_batched(aw, z, state.active, w_pos, w_act, **tiered)
    zero = torch.zeros(d, dtype=torch.float32, device=dev)
    one = zero + 1.0
    local, _ = ops.grad_batched(ops.GRAD_MOMENTS, z, w_pos, zero, one, 1.0, 1.0)
    shaped, _ = ops.grad_batched(ops.GRAD_MOMENTS, y, w_pos, zero, one, 1.0, 1.0)
    m, sigma = m.clone(), sigma.clone()
    p_sigma, p_c = state.p_sigma.reshape(B, d).clone(), state.p_c.reshape(B, d).clone()
    k = new(B, 3)
    ops.cmaes_vector_update_batched(local, shaped, m, p_sigma, p_c, sigma, _consts(hp) if tiers is None else ladder.consts, state.csa_squared, k,
                                    steps=steps, tier=tier)
    C_new = ops.weighted_syrk_update_batched(y, w_act, k, C.contiguous(), u=p_c, out=new(B, d, d))
    return m, p_sigma, p_c, sigma, C_new


def _assigned_weights(f: torch.Tensor, maximize: bool, weights: torch.Tensor, real: Optional[torch.Tensor] = None) -> torch.Tensor:
    """weights[rank of f[b, i] in row b], best first: a stable sort, NaN the largest value (the order of rank_table_batched).
    With `real` (B, n) (a padded population), row b ranks only its real rows, in the same order, with its own weights[b] (B, n);
    its pad rows come after them, at zero weight."""
    B, n = f.shape
    order = torch.argsort(f, dim=-1, descending=maximize, stable=True)
    if real is not None:
        order = order.gather(-1, torch.argsort((~real).gather(-1, order).to(torch.int32), dim=-1, stable=True))
    ranks = torch.empty_like(order).scatter_(-1, order, torch.arange(n, device=f.device).expand(B, n).contiguous())
    if real is not None:
        return torch.where(real, weights.gather(-1, ranks), 0.0)
    return weights.to(f.device)[ranks]


def _h_sig(hp: CMAESHyperparameters, pnorm: torch.Tensor, d: int, steps) -> torch.Tensor:
    """CMAES._h_sig per item, with the generation counter `steps` (an int, or a tensor of per-item counters) before its increment."""
    if isinstance(hp.c_sigma, torch.Tensor):
        decay = 1 - (1 - hp.c_sigma).pow((2 * steps + 1).to(pnorm.dtype))
    elif isinstance(steps, torch.Tensor):
        decay = 1 - torch.full_like(pnorm, 1 - hp.c_sigma).pow((2 * steps + 1).to(pnorm.dtype))
    else:
        decay = 1 - (1 - hp.c_sigma) ** (2 * steps + 1)
    squared_sum = pnorm.pow(2.0) / decay
    return ((squared_sum / d) - 1 < 1 + 4.0 / (d + 1)).to(pnorm.dtype)


def _tell_torch(state, hp, B, n, d, m, sigma, C, y, z, f, steps, tiers=None) -> tuple:
    """The same stages as batched torch ops (CMAES's op-by-op generation: update_m ... update_C, cmaes.py:454-553), with the
    generation counter `steps` (an int, or per-item counters).  `tiers`: as in `_tell` (the constants become per-item tensors)."""
    real = None
    if tiers is None:
        aw = _assigned_weights(f, state.maximize, hp.weights)
    else:
        hp, weights, real = _tier_items(tiers, n)
        aw = _assigned_weights(f, state.maximize, weights, real)
    w_pos = torch.clamp_min(aw, 0.0)
    local = torch.einsum("bn,bnd->bd", w_pos, z)
    shaped = torch.einsum("bn,bnd->bd", w_pos, y)
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
    w = torch.where(aw > 0, aw, d * aw / torch.sum(z * z, dim=-1)) if state.active else aw
    if real is not None:  # a pad row's 0 / ||0||^2
        w = torch.where(real, w, 0.0)
    c1a = hp.c_1 * (1 - (1 - h_sig**2) * hp.c_c * (2 - hp.c_c))
    pc = ((hp.c_1 / (c1a + 1e-23)) ** 0.5)[:, None] * p_c
    r1 = c1a[:, None, None] * (pc[:, :, None] * pc[:, None, :] - C)
    rmu = _col(hp.c_mu, 2) * ((y.mT * w[:, None, :]) @ y - _col(hp.weights_sum, 2) * C)
    return m, p_sigma, p_c, sigma, C + r1 + rmu
