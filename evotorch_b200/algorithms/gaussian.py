"""PGPE / SNES / CEM / XNES: search algorithms driven by a Gaussian search distribution (mirrors
evotorch.algorithms.distributed.gaussian, gaussian.py:35-1405: same constructor arguments, defaults and status keys).

One generation, as in the reference (gaussian.py:351-367): the gradient is computed from the population stored by the
PREVIOUS step, the distribution is updated, then a fresh population is sampled into the same buffers and evaluated.
For a CUDA float32 problem that is five kernel groups per generation and no host synchronisation:

    K3 rank -> K4 weighted column reduction -> K5 mu step -> K5 sigma step -> K1+K2 fused sample/evaluate

`distributed=True` shards the population over the ranks of torch.distributed (see ..distributed) instead of Ray actors.
"""

from __future__ import annotations

import math
import os
from copy import deepcopy
from typing import Optional

import torch

from .. import ops
from ..core import LazySolutionBatch, PhiloxSamples, Problem, SolutionBatch
from ..distributed import world
from ..distributions import Distribution, ExpGaussian, ExpSeparableGaussian, SeparableGaussian, SymmetricSeparableGaussian
from ..optimizers import get_optimizer_class
from ..tools.misc import modify_tensor, to_stdev_init
from .cudagraph import GenerationGraph
from .searchalgorithm import CUDAGraphMixin, SearchAlgorithm, SinglePopulationAlgorithmMixin


class GaussianSearchAlgorithm(SearchAlgorithm, SinglePopulationAlgorithmMixin, CUDAGraphMixin):
    """Base class of the Gaussian-distribution searchers (gaussian.py:35-501)."""

    DISTRIBUTION_TYPE = NotImplemented
    DISTRIBUTION_PARAMS = NotImplemented

    def __init__(self, problem: Problem, *, popsize: int, center_learning_rate: float, stdev_learning_rate: float,
                 stdev_init=None, radius_init=None, num_interactions: Optional[int] = None, popsize_max: Optional[int] = None,
                 optimizer=None, optimizer_config: Optional[dict] = None, ranking_method: Optional[str] = None, center_init=None,
                 stdev_min=None, stdev_max=None, stdev_max_change=None, obj_index: Optional[int] = None, distributed: bool = False,
                 popsize_weighted_grad_avg: Optional[bool] = None, ensure_even_popsize: bool = False):
        problem.ensure_numeric()
        problem.ensure_unbounded()
        SearchAlgorithm.__init__(self, problem, center=self._get_mu, stdev=self._get_sigma, mean_eval=self._get_mean_eval)
        # adaptive population size (gaussian.py:114-130, :299-349 of the reference): keep sampling `popsize`-sized populations until
        # the problem has reported more than `num_interactions` simulator interactions (or `popsize_max` solutions)
        self._num_interactions = None if num_interactions is None else int(num_interactions)
        if popsize_max is not None and num_interactions is None:
            raise ValueError("`popsize_max` was expected as None, because `num_interactions` is None."
                             " The argument `popsize_max` is meaningful only when `num_interactions` is given.")
        self._popsize_max = None if popsize_max is None else int(popsize_max)
        self._ensure_even_popsize = bool(ensure_even_popsize)
        if self._ensure_even_popsize and (int(popsize) % 2) != 0 and not distributed:
            raise ValueError(f"`popsize` was expected as an even number. However, the received `popsize` is {popsize}.")

        if center_init is None:
            mu = problem.generate_values(1).reshape(-1)
        else:
            mu = problem.ensure_tensor_length_and_dtype(center_init, allow_scalar=False, about="center_init").clone()
        stdev_init = to_stdev_init(solution_length=problem.solution_length, stdev_init=stdev_init, radius_init=radius_init)
        sigma = problem.ensure_tensor_length_and_dtype(stdev_init, about="stdev_init", allow_scalar=False).clone()

        dist_params = deepcopy(self.DISTRIBUTION_PARAMS) if self.DISTRIBUTION_PARAMS is not None else {}
        dist_params.update({"mu": mu, "sigma": sigma})
        self._distribution: Distribution = self.DISTRIBUTION_TYPE(dist_params, dtype=problem.dtype, device=problem.device)

        self._popsize = int(popsize)
        self._center_learning_rate = float(center_learning_rate)
        self._stdev_learning_rate = float(stdev_learning_rate)
        self._optimizer = self._initialize_optimizer(self._center_learning_rate, optimizer, optimizer_config)
        self._ranking_method = None if ranking_method is None else str(ranking_method)

        def bound(x, about):
            return None if x is None else problem.ensure_tensor_length_and_dtype(x, about=about, allow_scalar=True)

        self._stdev_min = bound(stdev_min, "stdev_min")
        self._stdev_max = bound(stdev_max, "stdev_max")
        self._stdev_max_change = bound(stdev_max_change, "stdev_max_change")

        def host_side(x):  # scalar bounds as python floats (read once here: no device->host sync per generation)
            return None if x is None else (float(x) if x.ndim == 0 else x)

        self._kernel_bounds = dict(lb=host_side(self._stdev_min), ub=host_side(self._stdev_max), max_change=host_side(self._stdev_max_change))
        self._obj_index = problem.normalize_obj_index(obj_index)

        # `distributed=True` shards the population over torch.distributed ranks (the reference needs Ray actors for this)
        self._distributed = bool(distributed) and world()[1] > 1
        self._step = self._step_distributed if self._distributed else self._step_non_distributed
        if popsize_weighted_grad_avg is not None and not distributed:
            raise ValueError("The argument `popsize_weighted_grad_avg` can only be used in distributed mode.")

        self._mean_eval = None
        self._population: Optional[SolutionBatch] = None
        self._first_iter = True
        CUDAGraphMixin.__init__(self)
        SinglePopulationAlgorithmMixin.__init__(self, exclude="mean_eval", enable=(not self._distributed))

    def _initialize_optimizer(self, learning_rate: float, optimizer=None, optimizer_config: Optional[dict] = None):
        if optimizer is None:
            return None
        if isinstance(optimizer, str):
            cls = get_optimizer_class(optimizer, optimizer_config)
            return cls(stepsize=float(learning_rate), dtype=self._distribution.dtype, solution_length=self._distribution.solution_length,
                       device=self._distribution.device)
        return optimizer

    # ------------------------------------------------------------------ generations
    def _fill_and_eval_pop(self):
        if self._num_interactions is not None:
            self._fill_and_eval_adaptive_pop()
            return
        if self._population is None:
            if self.problem.lazy_population:
                self._population = LazySolutionBatch(self.problem, self._popsize, device=self._distribution.device)
            else:
                self._population = SolutionBatch(self.problem, popsize=self._popsize, device=self._distribution.device, empty=True)
        self.problem.sample_and_evaluate(self._distribution, self._population)

    def _fill_and_eval_adaptive_pop(self):
        """gaussian.py:299-349: populations of `popsize` solutions are sampled and evaluated (each through the same fused K1+K2
        path as a fixed-size population) until the interaction count reported by the problem (`status["total_interaction_count"]`)
        has grown by more than `num_interactions`, or `popsize_max` solutions exist; the generation's population is their
        concatenation.  The population size then varies between generations, so this mode is never graph-captured."""
        prob = self.problem
        first = prob.status.get("total_interaction_count", 0)
        populations, total = [], 0
        while True:
            newpop = SolutionBatch(prob, popsize=self._popsize, device=self._distribution.device, empty=True)
            total += len(newpop)
            prob.sample_and_evaluate(self._distribution, newpop)
            populations.append(newpop)
            if self._popsize_max is not None and total >= self._popsize_max:
                break
            if prob.status["total_interaction_count"] - first > self._num_interactions:
                break
        self._population = populations[0] if len(populations) == 1 else SolutionBatch.cat(populations)

    # ------------------------------------------------------------------ CUDA-graph replay of a whole generation
    def _graph_capturable(self) -> bool:
        from ..optimizers import ClipUp

        dist, prob = self._distribution, self.problem
        ok = (self._num_interactions is None and isinstance(dist, SeparableGaussian) and ops.uses_kernels(dist.mu) and prob.rng == "philox"
              and prob.evok_objective_id is not None and len(prob.senses) == 1 and prob.eval_data_length == 0
              and (self._optimizer is None or isinstance(self._optimizer, ClipUp))
              and len(prob.before_eval_hook) == 0)  # a Python hook between sampling and evaluation cannot be replayed
        if self._distributed:  # the sharded generation has no Python between its kernels / collectives either
            return (ok and not prob.stores_solution_stats and len(prob.before_eval_hook) == 0 and len(prob.after_eval_hook) == 0
                    and len(prob.before_grad_hook) == 0 and len(prob.after_grad_hook) == 0)  # Python hooks do not replay
        return ok and self._population is not None

    def _graph_body(self):
        dist, prob, pop = self._distribution, self.problem, self._population
        lazy = isinstance(pop, LazySolutionBatch)
        n = len(pop)
        fitnesses = pop._evdata.view(-1)
        draw = prob.next_philox_draw()
        # the population consumed here is the previous generation's (the eager step before the capture, or the previous replay);
        # a materialised one is rebuilt in part from the same counters (`_step_graph` drops the graph if it was modified)
        recipe = draw.between_generations().recipe(n, dist.SYMMETRIC, dist.mu, dist.sigma)
        samples = recipe if lazy else PhiloxSamples(pop._data, recipe)
        gradients = dist.compute_gradients(samples, fitnesses, objective_sense=prob.senses[self._obj_index], ranking_method=self._ranking_method)
        self._update_into(dist.mu, dist.sigma, gradients)
        ops.sample_eval(prob.evok_objective_id, None if lazy else pop._data, dist.mu, dist.sigma, n_rows=n, symmetric=dist.SYMMETRIC,
                        f=fitnesses, **draw.kwargs)
        if lazy:
            pop.recipe = recipe

    def _step_graph(self):
        pop = self._population
        if self._graph is not None and self._graph_values_version is not None and pop._data._version != self._graph_values_version:
            # the population was modified in place since the last replay: the graph would rebuild rows from their Philox
            # counters, so this generation runs eagerly (reading the modified rows) and the next one captures a new graph
            self._graph = None
            self._step_eager()
            return
        if self._graph is None:
            # one more eager generation right before the capture: warms every kernel and workspace that the graph will use
            self._step_eager()
            # the distribution's tensors become the persistent, in-place-updated buffers of the graph
            dist, pop = self._distribution, self._population
            if not (dist.mu.is_contiguous() and dist.sigma.is_contiguous()):
                self._distribution = dist.modified_copy(mu=dist.mu.contiguous(), sigma=dist.sigma.contiguous())
            self._graph = GenerationGraph(self.problem, self._graph_body)
            # replays resample the population without passing through Python: the eager record goes stale with the first one
            pop._philox_record = None
            self._graph_values_version = None if isinstance(pop, LazySolutionBatch) else pop._data._version
            return
        self._graph.replay()
        self.problem._finish_evaluation(pop)

    def _step_non_distributed(self):
        """gaussian.py:274-367."""
        if self._first_iter:
            self._fill_and_eval_pop()
            self._first_iter = False
            return
        if self._use_graph and self._graph_capturable():
            self._step_graph()
        else:
            self._graph = None
            self._step_eager()

    def _step_eager(self):
        dist = self._distribution
        samples = self._population.gradient_samples(dist.mu, dist.sigma)
        fitnesses = self._population.access_evals()[:, self._obj_index]
        gradients = self._distribution.compute_gradients(samples, fitnesses, objective_sense=self.problem.senses[self._obj_index],
                                                         ranking_method=self._ranking_method)
        self._update_distribution(gradients)
        self._fill_and_eval_pop()

    def _distributed_body(self, in_place: bool):
        fetched = self.problem.sample_and_compute_gradients(self._distribution, self._popsize, obj_index=self._obj_index,
                                                            num_interactions=self._num_interactions, popsize_max=self._popsize_max,
                                                            ranking_method=self._ranking_method,
                                                            ensure_even_popsize=self._ensure_even_popsize)
        if in_place:
            self._update_into(self._distribution.mu, self._distribution.sigma, fetched[0]["gradients"])
        else:
            self._update_distribution(fetched[0]["gradients"])
        self._mean_eval = fetched[0]["mean_eval"]

    def _sync_initial_state(self):
        """First sharded generation: every rank adopts rank 0's distribution and optimizer state (replicated-update invariant;
        with center_init=None / seed=None the ranks would otherwise start from different centres and keep a constant offset)."""
        from ..distributed import broadcast_search_state

        dist_ = self._distribution
        tensors = [v for v in dist_.parameters.values() if isinstance(v, torch.Tensor)]
        opt = self._optimizer
        for name in ("_velocity", "_m", "_v", "_buf"):
            t = getattr(opt, name, None) if opt is not None else None
            if isinstance(t, torch.Tensor):
                tensors.append(t)
        broadcast_search_state(tensors)
        self._state_synced = True

    def _step_distributed(self):
        """Every rank: sample/evaluate its shard, global ranking, all-reduced gradients, replicated update
        (replaces gaussian.py:199-272).  With `enable_cuda_graph()` the whole sequence, NCCL collectives included, is captured
        once and replayed.  NOTE: replayed collectives run on the replaying stream, eager ones on NCCL's internal stream; do not
        interleave a graph-mode searcher with other collectives on the same process group without a device synchronisation."""
        prob = self.problem
        if not self.__dict__.get("_state_synced", False):
            self._sync_initial_state()
        if os.environ.get("EVOTORCH_B200_PEER", "0") == "1" and getattr(prob, "_peer_exchange", None) is None and not self.__dict__.get("_peer_tried"):
            # opt-in by environment: fuse the two exchanges of the generation into the producing kernels (evotorch_b200/peer.py)
            self._peer_tried = True
            from ..distributed import world
            from ..peer import enable_peer_exchange

            if world()[1] > 1 and ops.uses_kernels(self._distribution.mu) and prob.evok_objective_id is not None and prob.rng == "philox":
                enable_peer_exchange(prob, self._popsize)
        if not (self._use_graph and self._graph_capturable()):
            self._graph = None
            self._distributed_body(in_place=False)
            return
        if self._graph is None:
            if self._steps_count < 2:  # eager generations first: seed broadcast, NCCL communicators, workspaces, kernel warm-up
                self._distributed_body(in_place=False)
                return
            dist = self._distribution
            self._distribution = dist.modified_copy(mu=dist.mu.contiguous().clone(), sigma=dist.sigma.contiguous().clone())
            self._graph = GenerationGraph(prob, lambda: self._distributed_body(in_place=True))
        self._graph.replay()

    # ------------------------------------------------------------------ distribution update (K5)
    def _update_into(self, mu: torch.Tensor, sigma: torch.Tensor, gradients: dict):
        """The CUDA update of a separable distribution as two launches that write into `mu` and `sigma`: follow the gradients,
        then clamp sigma against its pre-update value."""
        gmu = gradients["mu"].contiguous()
        if self._optimizer is not None and hasattr(self._optimizer, "ascent_into_"):
            self._optimizer.ascent_into_(gmu, mu)
        elif self._optimizer is not None:
            mu += self._optimizer.ascent(gmu)
        else:
            ops.axpy_(mu, gmu, self._center_learning_rate)
        ops.sigma_update_(sigma, gradients["sigma"].contiguous(), self._stdev_learning_rate, isinstance(self._distribution, ExpSeparableGaussian),
                          **self._kernel_bounds)

    def _update_distribution(self, gradients: dict):
        """gaussian.py:369-419: follow the gradients, then clamp sigma against its pre-update value."""
        dist = self._distribution
        separable = isinstance(dist, SeparableGaussian)
        if separable and ops.uses_kernels(dist.mu) and ops.uses_kernels(gradients["mu"]):
            # on copies: the previous generation's tensors stay valid for whoever holds them
            new_mu, new_sigma = dist.mu.clone(), dist.sigma.clone()
            self._update_into(new_mu, new_sigma, gradients)
            self._distribution = dist.modified_copy(mu=new_mu, sigma=new_sigma)
            return

        controlled = (self._stdev_min is not None) or (self._stdev_max is not None) or (self._stdev_max_change is not None)
        old_sigma = dist.sigma if controlled else None
        learning_rates, optimizers = {}, {}
        if self._optimizer is not None:
            optimizers["mu"] = self._optimizer
        else:
            learning_rates["mu"] = self._center_learning_rate
        learning_rates["sigma"] = self._stdev_learning_rate
        updated = dist.update_parameters(gradients, learning_rates=learning_rates, optimizers=optimizers)
        if controlled:
            updated = updated.modified_copy(
                sigma=modify_tensor(old_sigma, updated.sigma, lb=self._stdev_min, ub=self._stdev_max, max_change=self._stdev_max_change))
        self._distribution = updated

    # ------------------------------------------------------------------ status
    def _get_mu(self) -> torch.Tensor:
        mu = self._distribution.parameters["mu"]
        return mu.clone() if self._graph is not None else mu  # graph replays update the live buffer in place

    def _get_sigma(self) -> torch.Tensor:
        sigma = self._distribution.parameters["sigma"]
        return sigma.clone() if self._graph is not None else sigma

    def _get_mean_eval(self) -> Optional[float]:
        if self._population is None:
            return None if self._mean_eval is None else float(self._mean_eval)
        return float(torch.mean(self._population.evals[:, self._obj_index]))

    @property
    def optimizer(self):
        """The center optimizer (`None`, `ClipUp`, `Adam` or `SGD`); `optimizer.param_groups[0]["lr"]` is readable/writable."""
        return None if self._optimizer is None else self._optimizer.contained_optimizer

    @property
    def population(self) -> Optional[SolutionBatch]:
        """The current population (None in sharded mode, where each rank only holds its shard)."""
        return self._population

    @property
    def obj_index(self) -> int:
        return self._obj_index


class PGPE(GaussianSearchAlgorithm):
    """Policy Gradients with Parameter-based Exploration (gaussian.py:503-744): symmetric sampling, ClipUp, centered
    ranking and stdev_max_change=0.2 by default."""

    DISTRIBUTION_TYPE = NotImplemented
    DISTRIBUTION_PARAMS = NotImplemented

    def __init__(self, problem: Problem, *, popsize: int, center_learning_rate: float, stdev_learning_rate: float, stdev_init=None,
                 radius_init=None, num_interactions: Optional[int] = None, popsize_max: Optional[int] = None, optimizer="clipup",
                 optimizer_config: Optional[dict] = None, ranking_method: Optional[str] = "centered", center_init=None, stdev_min=None,
                 stdev_max=None, stdev_max_change=0.2, symmetric: bool = True, obj_index: Optional[int] = None,
                 distributed: bool = False, popsize_weighted_grad_avg: Optional[bool] = None):
        if symmetric:
            self.DISTRIBUTION_TYPE = SymmetricSeparableGaussian
            divide_by = "num_directions"
        else:
            self.DISTRIBUTION_TYPE = SeparableGaussian
            divide_by = "num_solutions"
        self.DISTRIBUTION_PARAMS = {"divide_mu_grad_by": divide_by, "divide_sigma_grad_by": divide_by}
        super().__init__(problem, popsize=popsize, center_learning_rate=center_learning_rate, stdev_learning_rate=stdev_learning_rate,
                         stdev_init=stdev_init, radius_init=radius_init, popsize_max=popsize_max, num_interactions=num_interactions,
                         optimizer=optimizer, optimizer_config=optimizer_config, ranking_method=ranking_method, center_init=center_init,
                         stdev_min=stdev_min, stdev_max=stdev_max, stdev_max_change=stdev_max_change, obj_index=obj_index,
                         distributed=distributed, popsize_weighted_grad_avg=popsize_weighted_grad_avg, ensure_even_popsize=symmetric)


def _default_popsize(n: int) -> int:
    return int(4 + math.floor(3 * math.log(n)))


class SNES(GaussianSearchAlgorithm):
    """Separable Natural Evolution Strategies (gaussian.py:746-984): popsize 4+floor(3 ln n), lr_sigma 0.2(3+ln n)/sqrt(n)."""

    DISTRIBUTION_TYPE = ExpSeparableGaussian
    DISTRIBUTION_PARAMS = None

    def __init__(self, problem: Problem, *, stdev_init=None, radius_init=None, popsize: Optional[int] = None,
                 center_learning_rate: Optional[float] = None, stdev_learning_rate: Optional[float] = None,
                 scale_learning_rate: bool = True, num_interactions: Optional[int] = None, popsize_max: Optional[int] = None,
                 optimizer=None, optimizer_config: Optional[dict] = None, ranking_method: Optional[str] = "nes", center_init=None,
                 stdev_min=None, stdev_max=None, stdev_max_change=None, obj_index: Optional[int] = None, distributed: bool = False,
                 popsize_weighted_grad_avg: Optional[bool] = None):
        n = problem.solution_length
        if popsize is None:
            popsize = _default_popsize(n)
        if center_learning_rate is None:
            center_learning_rate = 1.0
        default_lr = 0.2 * (3 + math.log(n)) / math.sqrt(n)
        if stdev_learning_rate is None:
            stdev_learning_rate = default_lr
        else:
            stdev_learning_rate = float(stdev_learning_rate) * (default_lr if scale_learning_rate else 1.0)
        super().__init__(problem, popsize=popsize, center_learning_rate=center_learning_rate, stdev_learning_rate=stdev_learning_rate,
                         stdev_init=stdev_init, radius_init=radius_init, popsize_max=popsize_max, num_interactions=num_interactions,
                         optimizer=optimizer, optimizer_config=optimizer_config, ranking_method=ranking_method, center_init=center_init,
                         stdev_min=stdev_min, stdev_max=stdev_max, stdev_max_change=stdev_max_change, obj_index=obj_index,
                         distributed=distributed, popsize_weighted_grad_avg=popsize_weighted_grad_avg)


class CEM(GaussianSearchAlgorithm):
    """Cross-Entropy Method (gaussian.py:986-1181): the new distribution is the mean / std of the elite solutions."""

    DISTRIBUTION_TYPE = SeparableGaussian
    DISTRIBUTION_PARAMS = NotImplemented

    def __init__(self, problem: Problem, *, popsize: int, parenthood_ratio: float, stdev_init=None, radius_init=None,
                 num_interactions: Optional[int] = None, popsize_max: Optional[int] = None, center_init=None, stdev_min=None,
                 stdev_max=None, stdev_max_change=None, obj_index: Optional[int] = None, distributed: bool = False,
                 popsize_weighted_grad_avg: Optional[bool] = None):
        self.DISTRIBUTION_PARAMS = {"parenthood_ratio": float(parenthood_ratio)}
        super().__init__(problem, popsize=popsize, center_learning_rate=1.0, stdev_learning_rate=1.0, stdev_init=stdev_init,
                         radius_init=radius_init, popsize_max=popsize_max, num_interactions=num_interactions, optimizer=None,
                         optimizer_config=None, ranking_method=None, center_init=center_init, stdev_min=stdev_min, stdev_max=stdev_max,
                         stdev_max_change=stdev_max_change, obj_index=obj_index, distributed=distributed,
                         popsize_weighted_grad_avg=popsize_weighted_grad_avg)


class XNES(GaussianSearchAlgorithm):
    """Exponential Natural Evolution Strategies with a full covariance factor (gaussian.py:1183-1405)."""

    DISTRIBUTION_TYPE = ExpGaussian
    DISTRIBUTION_PARAMS = None

    def __init__(self, problem: Problem, *, stdev_init=None, radius_init=None, popsize: Optional[int] = None,
                 center_learning_rate: Optional[float] = None, stdev_learning_rate: Optional[float] = None,
                 scale_learning_rate: bool = True, num_interactions: Optional[int] = None, popsize_max: Optional[int] = None,
                 optimizer=None, optimizer_config: Optional[dict] = None, ranking_method: Optional[str] = "nes", center_init=None,
                 obj_index: Optional[int] = None, distributed: bool = False, popsize_weighted_grad_avg: Optional[bool] = None):
        n = problem.solution_length
        if popsize is None:
            popsize = _default_popsize(n)
        if center_learning_rate is None:
            center_learning_rate = 1.0
        default_lr = 0.6 * (3 + math.log(n)) / (n * math.sqrt(n))
        if stdev_learning_rate is None:
            stdev_learning_rate = default_lr
        else:
            stdev_learning_rate = float(stdev_learning_rate) * (default_lr if scale_learning_rate else 1.0)
        super().__init__(problem, popsize=popsize, center_learning_rate=center_learning_rate, stdev_learning_rate=stdev_learning_rate,
                         stdev_init=stdev_init, radius_init=radius_init, popsize_max=popsize_max, num_interactions=num_interactions,
                         optimizer=optimizer, optimizer_config=optimizer_config, ranking_method=ranking_method, center_init=center_init,
                         stdev_min=None, stdev_max=None, stdev_max_change=None, obj_index=obj_index, distributed=distributed,
                         popsize_weighted_grad_avg=popsize_weighted_grad_avg)
