"""Built-in vectorised objective functions with a fused evaluation kernel.

Each object is an ordinary vectorised fitness function (call it with an N x D tensor, get N fitnesses; it is marked
`__evotorch_vectorized__` like functions decorated with the reference's `@vectorized`, decorators.py:549) and
additionally carries `evok_objective_id`.  When a Problem is built around one of them, the Gaussian searchers
evaluate the population *inside* the sampling kernel (K1+K2 fused, csrc/evok_sample_eval.cu) so the N x D matrix is
written once and never re-read for evaluation.  Called directly on a CUDA fp32 population they run the stand-alone
row-reduction kernel (K2); on any other tensor the plain torch expression (same formula as the reference's README
example, README.md:86-89).

`FusedObjective` is the same for a user-defined function of sums over the elements (sum-separable) or over the neighbour
pairs (x_j, x_{j+1}) of a row (Rosenbrock, Trid, Dixon-Price): its expressions are compiled at run time into the same kernels
(evotorch_b200/jit.py), so every fused path of the package takes it.
"""

from __future__ import annotations

import math
from typing import Callable

import torch

from . import ops


class BuiltinObjective:
    __evotorch_vectorized__ = True

    def __init__(self, name: str, objective_id: int, torch_fn: Callable):
        self.__name__ = name
        self.name = name
        self.evok_objective_id = objective_id
        self._torch_fn = torch_fn

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if x.ndim == 1:
            return self._torch_fn(x.unsqueeze(0))[0]
        if ops.uses_kernels(x) and x.ndim == 2 and x.stride(1) == 1:
            return ops.evaluate(self.evok_objective_id, x)
        return self._torch_fn(x)

    def __repr__(self) -> str:
        return f"<evotorch_b200.objectives.{self.name}>"


def _sphere(x: torch.Tensor) -> torch.Tensor:
    return torch.sum(x**2, dim=-1)


def _rastrigin(x: torch.Tensor) -> torch.Tensor:
    n = x.shape[-1]
    return 10 * n + torch.sum((x**2) - 10 * torch.cos(2 * math.pi * x), dim=-1)


def _ackley(x: torch.Tensor) -> torch.Tensor:
    n = x.shape[-1]
    return (-20.0 * torch.exp(-0.2 * torch.sqrt(torch.sum(x**2, dim=-1) / n)) - torch.exp(torch.sum(torch.cos(2 * math.pi * x), dim=-1) / n)
            + 20.0 + math.e)


class FusedObjective(BuiltinObjective):
    """A user-defined objective f(x) = value(S_1, ..., S_k, D), k <= 4, fused into the sampler, where S_i is either
    sum_{j<D} term_i(x_j, j, D) or, for a term that uses xn = x_{j+1}, the pair sum sum_{j<D-1} term_i(x_j, x_{j+1}, j, D).

        styblinski_tang = FusedObjective("styblinski_tang", sums={"s": "x**4 - 16*x**2 + 5*x"}, value="0.5 * s")
        rosenbrock = FusedObjective("rosenbrock", sums={"s": "100*(xn - x**2)**2 + (1 - x)**2"}, value="s")

    `sums` maps each sum's name to its term (an expression of x, xn, j and D), `value` is an expression of the sums and D; the
    language is described in evotorch_b200.jit.  Construction parses both (ValueError for anything outside the language),
    compiles the kernels with NVRTC for sm_90a and registers them with libevok.so; `kernel_info` holds the registers and
    spills of every kernel.  The same source compiles once per process.  A FusedObjective pickles as its expressions.

    The batched samplers of the functional API (`pgpe_ask_and_evaluate`, `cem_ask_and_evaluate`) are 8 more kernels of the same
    source, compiled on the first batched use (`compile_batched`); `batched_kernel_info` then holds their registers and spills."""

    def __init__(self, name: str, sums: dict, value: str):
        from . import jit

        spec = jit.ObjectiveSpec(sums, value)
        if name in ops.OBJECTIVE_IDS and ops.OBJECTIVE_IDS[name] < ops.OBJ_USER_BASE:
            raise ValueError(f"{name!r} is the name of a built-in objective")
        compiled = jit.compile_objective(spec)
        super().__init__(name, compiled.objective_id, spec.torch_fn)
        self.sums, self.value, self.source = dict(spec.sums), spec.value, spec.source
        self.kernel_info = compiled.kernel_info
        self.batched_kernel_info = None
        self._spec = spec
        ops.OBJECTIVE_IDS[name] = compiled.objective_id

    def compile_batched(self) -> None:
        """Compile and attach the batched samplers (once per process for one source); fills `batched_kernel_info`."""
        if self.batched_kernel_info is None:
            from . import jit

            self.batched_kernel_info = jit.compile_batched(self._spec).kernel_info

    def __reduce__(self):
        return (FusedObjective, (self.name, self.sums, self.value))

    def __repr__(self) -> str:
        return f"FusedObjective({self.name!r}, sums={self.sums!r}, value={self.value!r})"


sphere = BuiltinObjective("sphere", ops.OBJ_SPHERE, _sphere)
rastrigin = BuiltinObjective("rastrigin", ops.OBJ_RASTRIGIN, _rastrigin)
ackley = BuiltinObjective("ackley", ops.OBJ_ACKLEY, _ackley)

__all__ = ["sphere", "rastrigin", "ackley", "BuiltinObjective", "FusedObjective"]
