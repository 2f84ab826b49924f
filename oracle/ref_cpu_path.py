"""The reference's CPU path for one PGPE generation, restated as the same sequence of torch CPU ops  --  TEST / BENCH
INFRASTRUCTURE ONLY (see oracle/es_oracle.py for the rules: never imported by the product).

Why this exists next to the numpy oracle: the reference IS a sequence of multi-threaded torch ops; timing a numpy port would
understate its speed.  `bench.py --impl reference` and the `cpu_baseline` leg therefore time THIS restatement with all host
threads (`kind: "port"`).  It is validated against the real reference's recorded runs in tests/golden (bit-identical trajectories,
tests/test_ref_cpu_port.py) and against the golden trajectories everywhere.

Op sequence per generation (gaussian.py:351-367 of the reference):
  rank         tools/ranking.py:44-53     argsort, arange/(n-1)-0.5, scatter
  gradients    distributions.py:708-773   X[0::2]-mu, (w+-w-)/2, row-scaled sums, /num_directions
  ClipUp       optimizers.py:309-357      g/|g|*lr, momentum, norm clip (host sync)
  sigma        distributions.py:591-596 + tools/misc.py:788-810 (modify_tensor with max_change)
  sample       tools/misc.py:1739-1749    strided normal_, copy, negate, *= sigma, += mu
  evaluate     README.md:86-89            10 n + sum(x^2 - 10 cos(2 pi x))
"""

from __future__ import annotations

import math
from typing import Optional

import torch


def rastrigin(x: torch.Tensor) -> torch.Tensor:
    n = x.shape[1]
    return 10 * n + torch.sum((x**2) - 10 * torch.cos(2 * math.pi * x), 1)


class PGPEReferencePath:
    """PGPE (symmetric, ClipUp, centered ranking, stdev_max_change) exactly as the reference's defaults run it on CPU."""

    def __init__(self, solution_length: int, popsize: int, *, center_learning_rate: float, stdev_learning_rate: float, stdev_init: float,
                 seed: int, stdev_max_change: Optional[float] = 0.2, momentum: float = 0.9, sense: str = "min",
                 center_init: Optional[torch.Tensor] = None, objective=rastrigin, device: str = "cpu"):
        # `device="cuda"` runs the very same torch op sequence on a GPU (the reference is device-agnostic): the "PyTorch eager
        # on the same GPU" comparator of SURVEY 8(d).  The CPU trajectory is what the golden tests pin.
        self.n, self.d = int(popsize), int(solution_length)
        self.device = torch.device(device)
        self.gen = torch.Generator(device=self.device).manual_seed(int(seed))
        if center_init is None:  # Problem.generate_values(1): uniform_() * (ub - lb) + lb  (core.py:1840-1909, tools/misc.py:1540)
            mu = torch.empty(1, self.d, device=self.device)
            mu.uniform_(generator=self.gen)
            mu *= torch.tensor(5.12) - torch.tensor(-5.12)
            mu += torch.tensor(-5.12)
            self.mu = mu.reshape(-1)
        else:
            self.mu = center_init.clone().to(self.device)
        self.sigma = torch.full((self.d,), float(stdev_init), device=self.device)
        self.lr, self.lr_sigma = float(center_learning_rate), float(stdev_learning_rate)
        self.momentum, self.max_speed = float(momentum), 2.0 * float(center_learning_rate)
        self.velocity = torch.zeros(self.d, device=self.device)
        self.max_change = stdev_max_change
        self.sense = sense
        self.objective = objective
        self.X = torch.empty(self.n, self.d, device=self.device)
        self.f: Optional[torch.Tensor] = None
        self.first = True

    def _sample_and_evaluate(self):
        out = self.X
        out[0::2, ...].normal_(generator=self.gen)
        out[1::2, ...] = out[0::2, ...]
        out[1::2, ...] *= -1
        out *= self.sigma
        out += self.mu
        self.f = self.objective(out)

    def _update(self):
        x, f = self.X, self.f
        n = len(f)
        indices = f.argsort(descending=(self.sense != "max"))
        weights = (torch.arange(n, dtype=f.dtype, device=f.device) / (n - 1)) - 0.5
        ranks = torch.empty_like(f)
        ranks[indices] = weights
        scaled_noises = x[0::2] - self.mu
        fdplus, fdminus = ranks[0::2], ranks[1::2]
        ndirs = n // 2
        grad_mu = torch.sum((((fdplus - fdminus) / 2) * scaled_noises.T).T, 0) / ndirs
        grad_sigma = torch.sum((((fdplus + fdminus) / 2) * (((scaled_noises**2) - (self.sigma**2)) / self.sigma).T).T, 0) / ndirs
        step = (grad_mu / torch.norm(grad_mu)) * self.lr
        v = (self.momentum * self.velocity) + step
        vnorm = torch.norm(v)
        if vnorm > self.max_speed:
            v = v * (self.max_speed / vnorm)
        self.velocity = v
        new_mu = self.mu + v.clone()
        new_sigma = self.sigma + self.lr_sigma * grad_sigma
        if self.max_change is not None:
            allowed = torch.abs(self.sigma) * torch.as_tensor(self.max_change, dtype=self.sigma.dtype)
            lb = torch.max(torch.as_tensor(float("-inf")), self.sigma - allowed)
            ub = torch.min(torch.as_tensor(float("inf")), self.sigma + allowed)
            new_sigma = torch.min(torch.max(new_sigma, lb), ub)
        self.mu, self.sigma = new_mu, new_sigma

    @torch.no_grad()
    def step(self):
        if self.first:
            self.first = False
        else:
            self._update()
        self._sample_and_evaluate()

    @property
    def mean_eval(self) -> float:
        return float(torch.mean(self.f))
