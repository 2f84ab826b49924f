"""Sample-and-evaluate for the functional ask / tell API: with the centre and stdev on the kernels and an objective that has a
fused kernel (`evok_objective_id`: the built-in objectives and every `FusedObjective`), the populations of all batch items are
drawn and evaluated in one launch of the batched sampler, which writes the population once and never reads it back for the
evaluation.  With `lazy=True` the population is not stored at all: the tell rebuilds the rows its gradient needs from their
Philox counters (`LazyPopulation`).

A `FusedObjective` whose data tensors have batch dimensions gives every batch item its own data, so one launch solves as many
problem instances as it has items.  The batch shape of the data is then the batch shape of the populations and fitnesses: the
centre and stdev are broadcast to it (`data_batch`).
"""

from __future__ import annotations

import math
from typing import Callable, Optional

import torch

from ... import ops
from ...objectives import is_transformed
from .misc import batch_shape_of, draw_philox_seed, flat_items, on_kernels


class LazyPopulation:
    """A population of shape (..., popsize, D) that was evaluated and not stored: the record of its draw (Philox seed, popsize,
    symmetric flag) and of the centre and stdev tensors it was drawn from (the tensors themselves and their `_version` at the
    draw).  `pgpe_tell` / `cem_tell` take it in place of the population; `materialize()` regenerates the population bit for bit.
    The tells rebuild the rows they need when their batch is the population's batch; when it is larger (batched hyper-parameters
    or fitnesses broadcast over the population's items) they materialise it for that tell, as a stored population is broadcast."""

    __slots__ = ("shape", "seed", "popsize", "symmetric", "center", "stdev", "center_version", "stdev_version")

    def __init__(self, shape: torch.Size, seed: int, popsize: int, symmetric: bool, center: torch.Tensor, stdev: torch.Tensor):
        self.shape = torch.Size(shape)
        self.seed, self.popsize, self.symmetric = int(seed), int(popsize), bool(symmetric)
        self.center, self.stdev = center, stdev
        self.center_version, self.stdev_version = center._version, stdev._version

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def check_drawn_from(self, center: torch.Tensor, stdev: torch.Tensor, symmetric: bool) -> None:
        """Raise ValueError unless the population was drawn from exactly these tensors, unmodified, with this symmetric flag
        (a host-side check: no device synchronisation)."""
        if center is not self.center or center._version != self.center_version:
            raise ValueError("this lazy population was drawn from another centre (or the centre was modified since): it can only be "
                             "told to the state it was asked from")
        if stdev is not self.stdev or stdev._version != self.stdev_version:
            raise ValueError("this lazy population was drawn from another stdev (or the stdev was modified since): it can only be "
                             "told to the state it was asked from")
        if bool(symmetric) != self.symmetric:
            raise ValueError(f"this lazy population was drawn with symmetric={self.symmetric}, the state samples with symmetric={symmetric}")

    def items(self) -> tuple:
        """(mu, sigma) as the batched kernels take them: (D,) when shared by every item, else (items, D)."""
        batch = self.shape[:-2]
        return (self.center if self.center.ndim == 1 else flat_items(self.center, batch, 1),
                self.stdev if self.stdev.ndim == 1 else flat_items(self.stdev, batch, 1))

    def materialize(self) -> torch.Tensor:
        """The population as a (..., popsize, D) tensor, bit-identical to the one a materialised ask would have stored."""
        self.check_drawn_from(self.center, self.stdev, self.symmetric)
        out = torch.empty(self.shape, dtype=self.center.dtype, device=self.center.device)
        mu, sigma = self.items()
        ops.sample_batched(out.view(-1, self.popsize, self.shape[-1]), mu, sigma, symmetric=self.symmetric, seed=self.seed)
        return out

    def __repr__(self) -> str:
        return f"LazyPopulation(shape={tuple(self.shape)}, seed={self.seed}, symmetric={self.symmetric})"


def fused_objective_id(objective: Callable, center: torch.Tensor, stdev: torch.Tensor) -> Optional[int]:
    """The objective id the batched sampler evaluates `objective` with, or None when the fused path does not apply (the centre
    or stdev is not a float32 CUDA tensor, or `objective` has no fused kernel)."""
    oid = getattr(objective, "evok_objective_id", None)
    if oid is None or oid == ops.OBJ_NONE or not on_kernels(center, stdev):
        return None
    if hasattr(objective, "compile_batched"):  # a FusedObjective: its batched kernels are compiled on the first batched use
        objective.compile_batched()
    return int(oid)


def data_batch(objective: Callable, batch: torch.Size) -> torch.Size:
    """The batch shape of a search whose centre and stdev have batch shape `batch` on `objective`: `batch` itself, or for an
    objective with per-item data the batch shape of the data, to which `batch` must broadcast (ValueError naming both if not)."""
    per_item = getattr(objective, "data_batch_shape", torch.Size())
    if not per_item:
        return batch
    try:
        ok = tuple(torch.broadcast_shapes(batch, per_item)) == tuple(per_item)
    except RuntimeError:
        ok = False
    if not ok:
        raise ValueError(f"the batch shape {tuple(batch)} of the centre and stdev does not broadcast to the batch shape {tuple(per_item)} "
                         f"of the data of {objective!r}")
    return per_item


def ask_and_evaluate_keyed(ask: Callable, batch: tuple, objective: Callable, searcher: str) -> tuple:
    """(values, evals) of a search whose ask is not the batched sampler's: `ask()` returns (values (*batch, popsize, D), the
    Philox seed of its draw, or None off the kernels).  With a seed, an objective with `evaluate_batched` and a kernel (a
    built-in objective or any FusedObjective, transformed and noisy ones included) evaluates every item in one call keyed with
    that seed, so a noisy objective gets the noise of the draw and per-item data gives item b its own data; otherwise this is
    `objective(values)`.  An objective whose data has a batch shape must have `batch` (ValueError naming `searcher` if not)."""
    per_item = tuple(getattr(objective, "data_batch_shape", ()))
    if per_item and per_item != tuple(batch):
        raise ValueError(f"the data of {objective!r} has batch shape {per_item}, the {searcher} state {tuple(batch)}: each item of the data "
                         "needs its own search (build the state with that batch shape)")
    values, seed = ask()
    oid = getattr(objective, "evok_objective_id", None)
    fused = (oid is not None and oid != ops.OBJ_NONE) or is_transformed(objective)
    if seed is not None and fused and hasattr(objective, "evaluate_batched"):
        return values, objective.evaluate_batched(values, seed=seed)
    return values, objective(values)


def ask_and_evaluate(ask: Callable, center: torch.Tensor, stdev: torch.Tensor, popsize: int, symmetric: bool, objective: Callable,
                     lazy: bool) -> tuple:
    """(population, fitnesses) of one ask: fused when `fused_objective_id` applies, else `ask()` followed by `objective`."""
    oid = fused_objective_id(objective, center, stdev)
    batch = data_batch(objective, batch_shape_of((center, 1), (stdev, 1)))
    if oid is None:
        if lazy:
            if is_transformed(objective):
                raise ValueError(f"lazy=True: {objective!r} reads the transformed row y = M (x - o), which needs the whole row; the fused "
                                 "sampler produces a row one column group at a time, so a transformed objective evaluates stored "
                                 "populations only (lazy=False)")
            oid = getattr(objective, "evok_objective_id", None)
            why = (f"{objective!r} has no fused kernel (use an objective of evotorch_b200.objectives or a FusedObjective)"
                   if oid is None or oid == ops.OBJ_NONE else "the centre and stdev are not float32 CUDA tensors")
            raise ValueError(f"lazy=True needs the fused sampler, which does not apply here: {why}")
        values = ask()
        return values.expand(tuple(batch) + values.shape[-2:]), objective(values)
    d = center.shape[-1]
    popsize = int(popsize)
    if symmetric and popsize % 2 != 0:
        raise ValueError(f"Symmetric sampling cannot be done if the number of solutions is odd: {popsize}")
    shape = torch.Size(tuple(batch) + (popsize, d))
    seed = draw_philox_seed()  # the draw of `ask()`: under the same torch.manual_seed the stored population is the asked one
    pop = LazyPopulation(shape, seed, popsize, symmetric, center, stdev)
    evals = torch.empty(shape[:-1], dtype=center.dtype, device=center.device)
    X = None if lazy else torch.empty(shape, dtype=center.dtype, device=center.device)
    mu, sigma = pop.items()
    n_items = math.prod(batch)
    ops.sample_eval_batched(oid, None if X is None else X.view(n_items, popsize, d), mu, sigma, evals.view(n_items, popsize),
                            symmetric=symmetric, seed=seed)
    return (pop if lazy else X), evals
