"""`NEProblem`: neuro-evolution problems whose solutions are the flat parameter vectors of a torch module (mirrors
evotorch.neuroevolution.neproblem.NEProblem, neproblem.py:33-429: same constructor arguments, `network_device`,
`network_constants`, `make_net`, `parameterize_net`, `_evaluate_network`, `_evaluate`).

The reference evaluates a population ONE SOLUTION AT A TIME: `_evaluate` fills the single instantiated network with a
solution's parameters (`parameterize_net`, neproblem.py:342-363) and calls the user's `network_eval_func` /
`_evaluate_network` on it (neproblem.py:407-429).  That contract -- an arbitrary Python function of an `nn.Module` -- is kept
as is.  What this class adds is the batched route for problems that can state their evaluation on the WHOLE population:
subclasses (or users) override `_evaluate_population(parameters) -> fitnesses`, where `parameters` is the N x L matrix of the
population (the storage the sampling kernel wrote), and use `self.batched_forward(parameters, x)`: row i of `parameters`
applied to a shared input batch `x` (B x in) -> N x B x out.  `SupervisedNE(common_minibatch=True)` is built on it; `VecNE` is
the B = 1-observation-per-policy case (K8).
"""

from __future__ import annotations

from copy import deepcopy
from typing import Any, Callable, Iterable, Optional, Union

import torch
from torch import nn

from ..core import Problem, Solution, SolutionBatch
from .policy import Policy, count_parameters, fill_parameters


def _pass_info_if_needed(fn: Callable, info: dict) -> Callable:
    """Functions decorated with @pass_info receive the problem's constants as keyword arguments (tools/misc.py `pass_info_if_needed`)."""
    if getattr(fn, "__evotorch_pass_info__", False):
        def wrapped(*args, **kwargs):
            merged = dict(info)
            merged.update(kwargs)
            return fn(*args, **merged)

        return wrapped
    return fn


class BaseNEProblem(Problem):
    """Common ancestor of the neuro-evolution problems (baseneproblem.py)."""


class NEProblem(BaseNEProblem):
    def __init__(self, objective_sense, network: Union[str, nn.Module, Callable[[], nn.Module]], network_eval_func: Optional[Callable] = None, *,
                 network_args: Optional[dict] = None, initial_bounds=(-0.00001, 0.00001), eval_dtype=None, eval_data_length: int = 0,
                 seed: Optional[int] = None, num_actors=None, actor_config: Optional[dict] = None, num_gpus_per_actor=None,
                 num_subbatches: Optional[int] = None, subbatch_size: Optional[int] = None, device=None):
        dev = torch.device("cpu" if device is None else device)
        self._original_network = network
        self._network_args = {} if network_args is None else deepcopy(network_args)
        if isinstance(self._original_network, nn.Module):
            self._original_network = self._original_network.cpu()
        self._network_eval_func: Optional[Callable] = network_eval_func
        self.instantiated_network: Optional[nn.Module] = None
        self._device = dev  # `network_device` is consulted while the temporary network is built
        temp_network = self._instantiate_net(self._original_network, device="cpu")
        super().__init__(objective_sense, initial_bounds=initial_bounds, solution_length=count_parameters(temp_network),
                         dtype=next(temp_network.parameters()).dtype, eval_dtype=eval_dtype, device=dev, eval_data_length=eval_data_length,
                         seed=seed, num_actors=num_actors, actor_config=actor_config, num_gpus_per_actor=num_gpus_per_actor,
                         num_subbatches=num_subbatches, subbatch_size=subbatch_size, store_solution_stats=None)
        self._policy: Optional[Policy] = None

    # ------------------------------------------------------------------ network construction (neproblem.py:251-340)
    @property
    def network_device(self) -> torch.device:
        """The device on which the problem places the network and its data (the problem's own device: there are no remote
        actors here, neproblem.py:251-261)."""
        return self._device

    @property
    def _str_network_constants(self) -> dict:
        """Named constants handed to `str_to_net`; override for problem-specific constants."""
        return {}

    @property
    def _network_constants(self) -> dict:
        """Named constants handed to the network's constructor; override for problem-specific constants."""
        return {}

    def network_constants(self) -> dict:
        constants = {}
        constants.update(self._network_constants)
        constants.update(self._network_args)
        return constants

    def _instantiate_net(self, network, device=None) -> nn.Module:
        if isinstance(network, str):
            from .net.parser import str_to_net

            consts = {}
            consts.update(self.network_constants())
            consts.update(self._str_network_constants)
            net = str_to_net(network, **consts)
        elif isinstance(network, nn.Module):
            net = network
        else:
            net = _pass_info_if_needed(network, self._network_constants)(**self._network_args)
        return net.to(self.network_device if device is None else device)

    def _prepare(self) -> None:
        self.instantiated_network = self._instantiate_net(self._original_network)
        self._original_network = None

    def _the_network(self) -> nn.Module:
        if self.instantiated_network is None:
            self.instantiated_network = self._instantiate_net(self._original_network)
        return self.instantiated_network

    def parameterize_net(self, parameters: torch.Tensor) -> nn.Module:
        """THE network of this problem, filled with `parameters` (neproblem.py:342-363)."""
        network = self._the_network()
        if parameters.device != self.network_device:
            parameters = parameters.to(self.network_device)
        fill_parameters(network, torch.as_tensor(parameters))
        return network

    def make_net(self, parameters: Iterable) -> nn.Module:
        """A NEW network filled with `parameters` (a Solution or anything convertible to a 1-D tensor) (neproblem.py:322-340)."""
        if isinstance(parameters, Solution):
            parameters = parameters.access_values(keep_evals=True)
        else:
            parameters = self.make_tensor(parameters)
        with torch.no_grad():
            return deepcopy(self.parameterize_net(parameters))

    @property
    def _grad_device(self) -> torch.device:
        return self.network_device

    # ------------------------------------------------------------------ evaluation
    def _evaluate_network(self, network: nn.Module) -> Union[float, torch.Tensor, tuple]:
        """Override point: fitness (scalar / 1-D tensor / (fitness, eval_data) tuple) of a parameterised network (neproblem.py:385-405)."""
        raise NotImplementedError

    def _evaluate(self, solution: Solution):
        """One solution: fill the network, call the evaluator (neproblem.py:407-429)."""
        evaluator = self._evaluate_network if self._network_eval_func is None else self._network_eval_func
        fitnesses = evaluator(self.parameterize_net(solution.values))
        if isinstance(fitnesses, tuple):
            solution.set_evals(*fitnesses)
        else:
            solution.set_evals(fitnesses)

    def _evaluate_population(self, parameters: torch.Tensor) -> Optional[Union[torch.Tensor, tuple]]:
        """Batched override point (not in the reference): fitnesses of ALL rows of the N x L parameter matrix at once, or None
        to fall back to the reference's one-solution-at-a-time loop."""
        return None

    def _evaluate_batch(self, batch: SolutionBatch):
        result = self._evaluate_population(batch.access_values(keep_evals=True))
        if result is None:
            for solution in batch:
                self._evaluate(solution)
        elif isinstance(result, tuple):
            batch.set_evals(*result)
        else:
            batch.set_evals(result)

    # ------------------------------------------------------------------ batched forward
    @property
    def policy(self) -> Policy:
        """The flat-parameter view of the network (`Policy`): recognises feed-forward nets for the kernel paths."""
        if self._policy is None:
            self._policy = Policy(self._the_network())
        return self._policy

    @torch.no_grad()
    def batched_forward(self, parameters: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
        """Row i of `parameters` (N x L) applied to the SHARED input batch `x` (B x ...) -> N x B x out.
        This is the one place where the policy forward of a population is a dense contraction: for a feed-forward net the first
        layer of all N networks is ONE product (N*H x in) * (in x B) of the stacked weight rows with the shared batch; on CUDA
        float32 it runs on the tensor-core GEMM kernel with the weights read once (`Policy.forward_shared`)."""
        return self.policy.forward_shared(parameters, x)

    def to_policy(self, solution) -> nn.Module:
        """A copy of the network carrying the parameters of `solution` (a Solution or a flat vector)."""
        return self.make_net(solution)
