"""CMA-ES with a full covariance matrix and active weights (mirrors evotorch.algorithms.cmaes.CMAES, cmaes.py:90-606:
same constructor arguments, hyper-parameter formulas and status keys).

Per generation (cmaes.py:567-606):
    z ~ N(0, I) (K1 Philox sampler on CUDA)  ->  Y = Z A^T, X = m + sigma*Y (one GEMM with the affine epilogue)
    evaluate (K2 for built-in objectives)  ->  stable argsort (K3)  ->  rank -> weight gather
    weighted recombinations sum_i w_i z_i, sum_i w_i y_i (K4 weighted column sums)
    evolution paths, sigma, rank-1 + rank-mu update of C, Cholesky.
The rank-mu term is computed as Y^T diag(w) Y (a weighted SYRK): the reference materialises an N x D x D broadcast
temporary (cmaes.py:548; 16 GiB at D = 1024, N = 4096).  On CUDA fp32 both contractions run on the hand-written wgmma
kernel (csrc/evok_gemm.cu: TMA -> 128B-swizzled smem -> wgmma.mma_async tf32 with 3xTF32 operand splitting -> registers ->
register accumulation; the lo halves of the 3xTF32 operands are derived inside the kernel, so operands are read from HBM once); the
glue between the contractions is fused into four small kernels (csrc/evok_cmaes.cu, evok_rank_table) and the covariance update is
applied by the SYRK's epilogue, so a generation is ~14 launches with no host reads and replays from a CUDA graph
(`enable_cuda_graph()`).  The Cholesky factorisation stays on cuSOLVER (torch.linalg.cholesky_ex): the repo's own persistent
tile-dataflow kernel (csrc/evok_chol.cu, EVOTORCH_B200_EVOK_CHOLESKY=1) is correct but its 64 x 64 diagonal tiles form a serial critical path.

Separable CMA-ES (`separable=True`, diagonal C) has its own fused generation on CUDA fp32 (`_step_sep_fused`): four kernels, no
host reads, the population written once (or never, with `Problem(lazy_population=True)`) and never read back, stdev bounds
included, CUDA-graph capturable at any `decompose_C_freq`.  The op-by-op path stays for CPU, rng="torch" and other dtypes.
"""

from __future__ import annotations

import math
import os
from typing import NamedTuple, Optional, Tuple

import numpy as np
import torch

from .. import ops
from ..core import LazySolutionBatch, Problem, Solution, SolutionBatch
from .cudagraph import GenerationGraph
from .searchalgorithm import CUDAGraphMixin, SearchAlgorithm, SinglePopulationAlgorithmMixin


def _safe_divide(a, b):
    tolerance = 1e-8
    if abs(b) < tolerance:
        b = (-tolerance) if b < 0 else tolerance
    return a / b


class CMAESHyperparameters(NamedTuple):
    """The recombination weights and learning rates of a CMA-ES search (see `cmaes_hyperparameters`)."""

    popsize: int
    mu: int
    weights: torch.Tensor
    weights_sum: float
    mu_eff: float
    c_m: float
    c_sigma: float
    damp_sigma: float
    c_c: float
    c_1: float
    c_mu: float
    variance_discount_sigma: float
    variance_discount_c: float
    unbiased_expectation: float
    decompose_C_freq: int


def cmaes_hyperparameters(d: int, popsize: Optional[int], *, dtype: torch.dtype, device, c_m: float = 1.0, c_sigma: Optional[float] = None,
                          c_sigma_ratio: float = 1.0, damp_sigma: Optional[float] = None, damp_sigma_ratio: float = 1.0, c_c: Optional[float] = None,
                          c_c_ratio: float = 1.0, c_1: Optional[float] = None, c_1_ratio: float = 1.0, c_mu: Optional[float] = None,
                          c_mu_ratio: float = 1.0, active: bool = True, separable: bool = False,
                          limit_C_decomposition: bool = True) -> CMAESHyperparameters:
    """Default population size, recombination weights and learning rates of CMA-ES for solution length `d` (cmaes.py:270-385 of the
    reference): host scalars in float64, the weight vector in `dtype` on `device`.  `CMAES` and the functional `cmaes` both take them
    from here."""
    if not popsize:
        popsize = 4 + int(np.floor(3 * np.log(d)))  # cmaes.py:270-272
    popsize = int(popsize)
    mu = int(np.floor(popsize / 2))
    raw_weights = torch.as_tensor(np.log((popsize + 1) / 2) - torch.log(torch.arange(popsize) + 1), dtype=dtype, device=device)
    positive, negative = raw_weights[:mu], raw_weights[mu:]
    mu_eff = float(torch.sum(positive).pow(2.0) / torch.sum(positive.pow(2.0)))
    if c_sigma is None:
        c_sigma = (mu_eff + 2.0) / (d + mu_eff + 3)
    c_sigma = c_sigma_ratio * c_sigma
    if damp_sigma is None:
        damp_sigma = 1 + 2 * max(0.0, math.sqrt((mu_eff - 1) / (d + 1)) - 1) + c_sigma
    damp_sigma = damp_sigma_ratio * damp_sigma
    if c_c is None:
        if separable:
            c_c = (1 + (1 / d) + (mu_eff / d)) / (d**0.5 + (1 / d) + 2 * (mu_eff / d))
        else:
            c_c = (4 + mu_eff / d) / (d + (4 + 2 * mu_eff / d))
    c_c = c_c_ratio * c_c
    if c_1 is None:
        if separable:
            c_1 = 1.0 / (d + 2.0 * np.sqrt(d) + mu_eff / d)
        else:
            c_1 = min(1, popsize / 6) * 2 / ((d + 1.3) ** 2.0 + mu_eff)
    c_1 = float(c_1_ratio * c_1)
    if c_mu is None:
        if separable:
            c_mu = (0.25 + mu_eff + (1.0 / mu_eff) - 2) / (d + 4 * np.sqrt(d) + (mu_eff / 2.0))
        else:
            c_mu = min(1 - c_1, 2 * ((0.25 + mu_eff - 2 + (1 / mu_eff)) / ((d + 2) ** 2.0 + mu_eff)))
    c_mu = float(c_mu_ratio * c_mu)
    positive = positive / torch.sum(positive)
    if active:
        mu_eff_neg = float(torch.sum(negative).pow(2.0) / torch.sum(negative.pow(2.0)))
        alpha = min(1 + c_1 / c_mu, 1 + 2 * mu_eff_neg / (mu_eff + 2), (1 - c_mu - c_1) / (d * c_mu))
        negative = alpha * negative / torch.sum(torch.abs(negative))
    else:
        negative = torch.zeros_like(negative)
    weights = torch.cat([positive, negative], dim=-1)
    if limit_C_decomposition:
        decompose_C_freq = max(1, int(np.floor(_safe_divide(1, 10 * d * (c_1 + c_mu)))))
    else:
        decompose_C_freq = 1
    return CMAESHyperparameters(popsize=popsize, mu=mu, weights=weights, weights_sum=float(torch.sum(weights)), mu_eff=mu_eff, c_m=c_m,
                                c_sigma=c_sigma, damp_sigma=damp_sigma, c_c=c_c, c_1=c_1, c_mu=c_mu,
                                variance_discount_sigma=math.sqrt(c_sigma * (2 - c_sigma) * mu_eff),
                                variance_discount_c=math.sqrt(c_c * (2 - c_c) * mu_eff),
                                unbiased_expectation=np.sqrt(d) * (1 - (1 / (4 * d)) + 1 / (21 * d**2)), decompose_C_freq=decompose_C_freq)


class CMAES(SearchAlgorithm, SinglePopulationAlgorithmMixin, CUDAGraphMixin):
    def __init__(self, problem: Problem, *, stdev_init, popsize: Optional[int] = None, center_init=None, c_m: float = 1.0,
                 c_sigma: Optional[float] = None, c_sigma_ratio: float = 1.0, damp_sigma: Optional[float] = None,
                 damp_sigma_ratio: float = 1.0, c_c: Optional[float] = None, c_c_ratio: float = 1.0, c_1: Optional[float] = None,
                 c_1_ratio: float = 1.0, c_mu: Optional[float] = None, c_mu_ratio: float = 1.0, active: bool = True,
                 csa_squared: bool = False, stdev_min: Optional[float] = None, stdev_max: Optional[float] = None,
                 separable: bool = False, limit_C_decomposition: bool = True, obj_index: Optional[int] = None):
        SearchAlgorithm.__init__(self, problem, center=self._get_center, stepsize=self._get_sigma)
        problem.ensure_numeric()
        problem.ensure_unbounded()
        self._obj_index = problem.normalize_obj_index(obj_index)
        d = problem.solution_length
        # weights and learning rates (cmaes.py:270-385)
        hp = cmaes_hyperparameters(d, popsize, dtype=problem.dtype, device=problem.device, c_m=c_m, c_sigma=c_sigma, c_sigma_ratio=c_sigma_ratio,
                                   damp_sigma=damp_sigma, damp_sigma_ratio=damp_sigma_ratio, c_c=c_c, c_c_ratio=c_c_ratio, c_1=c_1,
                                   c_1_ratio=c_1_ratio, c_mu=c_mu, c_mu_ratio=c_mu_ratio, active=active, separable=separable,
                                   limit_C_decomposition=limit_C_decomposition)
        popsize = self.popsize = hp.popsize
        self.mu = hp.mu
        self.separable = bool(separable)
        if self.separable and problem.lazy_population:
            # the fused separable generation never reads the population back, so it can stay a function of the Philox counters.
            # No initial values are drawn for it, so with center_init=None the random centre below differs from the one of a
            # materialised run with the same seed (whose initial population consumes the generator first, as in the reference).
            if not (problem.evok_objective_id is not None and problem.rng == "philox" and len(problem.senses) == 1
                    and problem.eval_data_length == 0 and problem.device.type == "cuda" and problem.dtype == torch.float32):
                raise ValueError("a lazy population needs a built-in objective, rng='philox', a separable Gaussian and CUDA float32")
            self._population = LazySolutionBatch(problem, popsize)
        else:
            self._population = problem.generate_batch(popsize=popsize)

        if center_init is None:
            center_init = problem.generate_values(1)
        elif isinstance(center_init, Solution):
            center_init = center_init.values.clone()
        # reshape, not squeeze: with solution_length 1 a squeezed (1, 1) centre would be a 0-d tensor and fail the check below
        self.m = problem.make_tensor(center_init).reshape(-1).clone()
        if not (self.m.ndim == 1 and len(self.m) == d):
            raise ValueError(f"The initial center point was expected as a vector of length {d}."
                             " However, the provided `center_init` has (or implies) a different shape.")
        self.sigma = problem.make_tensor(stdev_init)
        if separable:
            self.C = problem.make_ones(d)
            self.A = problem.make_ones(d)
        else:
            self.C = problem.make_I(d)
            self.A = self.C.clone()

        self.mu_eff, self.c_m, self.c_sigma, self.damp_sigma, self.c_c = hp.mu_eff, hp.c_m, hp.c_sigma, hp.damp_sigma, hp.c_c
        self.c_1, self.c_mu, self.variance_discount_sigma, self.variance_discount_c = hp.c_1, hp.c_mu, hp.variance_discount_sigma, hp.variance_discount_c
        self.weights, self._weights_sum, self.unbiased_expectation, self.decompose_C_freq = hp.weights, hp.weights_sum, hp.unbiased_expectation, hp.decompose_C_freq
        self.active, self.csa_squared = bool(active), bool(csa_squared)
        self.stdev_min, self.stdev_max = stdev_min, stdev_max
        self.p_sigma = problem.make_zeros(d)
        self.p_c = problem.make_zeros(d)
        CUDAGraphMixin.__init__(self)
        SinglePopulationAlgorithmMixin.__init__(self)

    # ------------------------------------------------------------------ accessors
    @property
    def population(self) -> SolutionBatch:
        return self._population

    @property
    def obj_index(self) -> int:
        return self._obj_index

    def _get_center(self) -> torch.Tensor:
        return self.m.clone() if self.__dict__.get("_fused") is not None else self.m  # the fused step updates `m` in place

    def _get_sigma(self) -> float:
        return float(self.sigma)

    # ------------------------------------------------------------------ one generation
    def sample_distribution(self, num_samples: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """zs ~ N(0, I); ys = zs A^T; xs = m + sigma ys (cmaes.py:408-430)."""
        n = self.popsize if num_samples is None else int(num_samples)
        problem = self._problem
        d = problem.solution_length
        # persistent buffers of the fused generation (the separable one draws inside its own sampler and keeps no zs)
        fs = self.__dict__.get("_fused") if n == self.popsize and not self.separable else None
        zs = problem.make_empty(num_solutions=n) if fs is None else fs["zs"]
        self.__dict__.pop("_z_draw", None)
        if ops.uses_kernels(zs) and problem.rng == "philox":
            zero, one = (problem.make_zeros(d), problem.make_ones(d)) if fs is None else (fs["zero"], fs["one"])
            draw = problem.next_philox_draw()
            ops.sample_eval(ops.OBJ_NONE, zs, zero, one, n_rows=n, symmetric=False, **draw.kwargs)
            # row i of xs is m + sigma A z_i of this draw: an objective with noise evaluates it with the same draw (_rows_draw)
            self._z_draw = draw
        else:
            problem.make_gaussian(out=zs)
        if self.separable:
            ys = self.A.unsqueeze(0) * zs
        elif ops.uses_kernels(zs) and ops.uses_kernels(self.A):
            # K6: one tensor-core GEMM (3xTF32, fp32-accurate) with the affine epilogue xs = m + sigma * ys fused in; in the fused
            # generation xs IS the population's value buffer
            ys = torch.empty_like(zs) if fs is None else fs["ys"]
            xs = torch.empty_like(zs) if fs is None else self._population._data
            ops.gemm_nt(zs, self.A.contiguous(), ys, out2=xs, alpha=self.sigma.reshape(1), bias=self.m.contiguous())
            return zs, ys, xs
        else:
            ys = zs @ self.A.T
        xs = self.m.unsqueeze(0) + self.sigma * ys
        return zs, ys, xs

    def _take_z_draw(self):
        """The z draw of the population about to be evaluated (taken once), or None: rows that a before-eval hook may edit, or that
        an overriding `sample_distribution` produced, have no draw of their own."""
        draw = self.__dict__.pop("_z_draw", None)
        if len(self._problem.before_eval_hook) or "sample_distribution" in self.__dict__ or type(self).sample_distribution is not CMAES.sample_distribution:
            return None
        return draw

    def get_population_weights(self, xs: torch.Tensor) -> torch.Tensor:
        """Evaluate, sort best-first, weight of each solution = weights[rank] (cmaes.py:432-452)."""
        self._population.set_values(xs)
        with self._problem._rows_drawn_by(self._take_z_draw()):
            self._problem.evaluate(self._population)
        indices = self._population.argsort(obj_index=self.obj_index)
        ranks = torch.empty_like(indices)
        ranks[indices] = torch.arange(self.popsize, dtype=indices.dtype, device=indices.device)
        return self.weights[ranks]

    def _weighted_rowsum(self, w: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
        """sum_i w_i rows_i -- K4 (moments form with a zero centre) on CUDA fp32."""
        if ops.uses_kernels(rows) and ops.uses_kernels(w):
            d = rows.shape[1]
            zero = torch.zeros(d, dtype=rows.dtype, device=rows.device)
            one = torch.ones(d, dtype=rows.dtype, device=rows.device)
            s1, _ = ops.grad(ops.GRAD_MOMENTS, rows.contiguous(), w.contiguous(), zero, one, 1.0, 1.0)
            return s1
        return torch.mv(rows.T, w)

    def update_m(self, zs, ys, assigned_weights) -> Tuple[torch.Tensor, torch.Tensor]:
        """Weighted recombination of the mu best (exactly the solutions with positive weight) (cmaes.py:454-481)."""
        positive = torch.clamp_min(assigned_weights, 0.0)
        local_m_displacement = self._weighted_rowsum(positive, zs)
        shaped_m_displacement = self._weighted_rowsum(positive, ys)
        self.m = self.m + self.c_m * self.sigma * shaped_m_displacement
        return local_m_displacement, shaped_m_displacement

    def update_p_sigma(self, local_m_displacement: torch.Tensor) -> None:
        self.p_sigma = (1 - self.c_sigma) * self.p_sigma + self.variance_discount_sigma * local_m_displacement

    def update_sigma(self) -> None:
        d = self._problem.solution_length
        if self.csa_squared:
            exponential_update = (torch.norm(self.p_sigma).pow(2.0) / d - 1) / 2
        else:
            exponential_update = torch.norm(self.p_sigma) / self.unbiased_expectation - 1
        self.sigma = self.sigma * torch.exp((self.c_sigma / self.damp_sigma) * exponential_update)

    def _h_sig(self) -> torch.Tensor:
        """cmaes.py:31-46 (uses the generation counter before it is incremented); stays a device scalar: no host sync."""
        d = self.p_sigma.shape[-1]
        squared_sum = torch.norm(self.p_sigma).pow(2.0) / (1 - (1 - self.c_sigma) ** (2 * self._steps_count + 1))
        return ((squared_sum / d) - 1 < 1 + 4.0 / (d + 1)).to(self.p_sigma.dtype)

    def update_p_c(self, shaped_m_displacement: torch.Tensor, h_sig: torch.Tensor) -> None:
        self.p_c = (1 - self.c_c) * self.p_c + h_sig * self.variance_discount_c * shaped_m_displacement

    def update_C(self, zs, ys, assigned_weights, h_sig) -> None:
        """Rank-1 + rank-mu update with active (negative) weights (cmaes.py:519-553)."""
        d = self._problem.solution_length
        if self.active:
            assigned_weights = torch.where(assigned_weights > 0, assigned_weights,
                                           d * assigned_weights / torch.sum(zs * zs, dim=-1))
        c1a = self.c_1 * (1 - (1 - h_sig**2) * self.c_c * (2 - self.c_c))
        weighted_pc = (self.c_1 / (c1a + 1e-23)) ** 0.5
        if self.separable:
            r1_update = c1a * (self.p_c.pow(2.0) - self.C)
            rmu_update = self.c_mu * (self._weighted_rowsum(assigned_weights, ys.pow(2.0)) - torch.sum(assigned_weights) * self.C)
        else:
            pc = weighted_pc * self.p_c
            r1_update = c1a * (torch.outer(pc, pc) - self.C)
            if ops.uses_kernels(ys) and ops.uses_kernels(assigned_weights):
                # K7: weighted SYRK Y^T diag(w) Y as one tensor-core GEMM over K-major (w*Y)^T and Y^T (split-K over the population)
                syrk = ops.gemm_nt(ops.transpose_scale(ys.contiguous(), assigned_weights.contiguous()), ops.transpose_scale(ys.contiguous()))
            else:
                syrk = (ys.T * assigned_weights) @ ys  # no N x D x D temporary either
            rmu_update = self.c_mu * (syrk - self._weights_sum * self.C)
        self.C = self.C + r1_update + rmu_update

    def _limit_stdev(self) -> None:
        """cmaes.py:49-79."""
        diag = self.C if self.separable else torch.diag(self.C)
        stdevs = torch.clamp(self.sigma * torch.sqrt(diag), min=self.stdev_min, max=self.stdev_max)
        unscaled = (stdevs / self.sigma).pow(2.0)
        if self.separable:
            self.C = unscaled
        else:
            self.C = self.C.clone()
            torch.diagonal(self.C)[:] = unscaled

    def decompose_C(self) -> None:
        if self.separable:
            self.A = self.C.pow(0.5)
        elif ops.uses_kernels(self.C) and self.C.is_contiguous() and os.environ.get("EVOTORCH_B200_EVOK_CHOLESKY", "0") == "1":
            self.A = ops.cholesky(self.C)
        else:
            self.A = torch.linalg.cholesky(self.C)

    # ------------------------------------------------------------------ fused generation (CUDA float32)
    def _fused_ok(self) -> bool:
        pop = self._population
        if self.separable:  # stdev bounds are applied by the update kernel; the sampler is built in, so an override stays op-by-op
            return (ops.uses_kernels(self.m) and ops.uses_kernels(self.C) and self._problem.rng == "philox"
                    and (isinstance(pop, LazySolutionBatch) or pop._data.is_contiguous()) and pop._evdata.shape[1] == 1
                    and pop._evdata.dtype == torch.float32 and "sample_distribution" not in self.__dict__
                    and type(self).sample_distribution is CMAES.sample_distribution)
        return (self.stdev_min is None and self.stdev_max is None and ops.uses_kernels(self.m) and ops.uses_kernels(self.C)
                and self._problem.rng == "philox" and pop._data.is_contiguous()
                and pop._evdata.shape[1] == 1 and pop._evdata.dtype == torch.float32)

    def _fused_state(self) -> dict:
        fs = self.__dict__.get("_fused")
        if fs is not None:
            return fs
        p, n, d, dev = self._problem, self.popsize, self._problem.solution_length, self.m.device
        new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)  # noqa: E731
        if self.separable:
            lazy = isinstance(self._population, LazySolutionBatch)
            # m_draw / s_draw: the centre and stdev the current (lazy) population was drawn from, written by the update kernel
            fs = dict(q=new(n), aw=new(n), local=new(d), S2=new(d), wsum=new(1), m_draw=new(d) if lazy else None, s_draw=new(d) if lazy else None)
        else:
            fs = dict(zs=new(n, d), ys=new(n, d), aw=new(n), w_pos=new(n), w_act=new(n), local=new(d), shaped=new(d), scratch=new(d), k=new(3),
                      zero=p.make_zeros(d), one=p.make_ones(d), info=torch.zeros((), dtype=torch.int32, device=dev))
        # state tensors become persistent buffers that the kernels update in place (pointer-stable: CUDA-graph replay)
        self.m, self.p_sigma, self.p_c = self.m.contiguous().clone(), self.p_sigma.contiguous().clone(), self.p_c.contiguous().clone()
        self.sigma = self.sigma.reshape(()).clone()
        self.C, self.A = self.C.contiguous().clone(), self.A.contiguous().clone()
        if self.separable:
            fs["s"] = (self.sigma * self.A).contiguous()  # the sampler's per-column stdev; the update kernel keeps it = sigma * A
        self._consts = (self.c_m, self.c_sigma, self.damp_sigma, self.c_c, self.c_1, self.c_mu, self.variance_discount_sigma,
                        self.variance_discount_c, float(self.unbiased_expectation), self._weights_sum)
        self._fused = fs
        return fs

    def _step_fused(self, steps_dev: Optional[torch.Tensor] = None):
        """One generation as a short chain of kernels with no host reads (cmaes.py:567-606):
        K1 z-sampling -> GEMM (Y = Z A^T, X = m + sigma Y straight into the population) -> evaluate -> rank-to-weights (K3, one launch)
        -> row weights (positive part / active reweighting, one pass over Z) -> two weighted row sums (K4) -> fused vector update
        (m, p_sigma, sigma, h_sig, p_c + the covariance coefficients) -> weighted SYRK with the covariance update in its epilogue ->
        Cholesky.  Every state tensor is updated in place.  Under a CUDA-graph capture `steps_dev` is the device-side step
        counter that the vector update reads and increments (`_h_sig`, the decomposition schedule); eager steps use `_steps_count`."""
        if self.separable:
            self._step_sep_fused(steps_dev)
            return
        fs = self._fused_state()
        zs, ys, xs = self.sample_distribution()
        pop = self._population
        if xs.data_ptr() == pop._data.data_ptr():
            pop._evdata.fill_(float("nan"))
        else:  # an overriding `sample_distribution` (e.g. recorded draws in the tests) returns its own tensors
            pop.set_values(xs)
        with self._problem._rows_drawn_by(self._take_z_draw()):
            self._problem.evaluate(pop)
        f = pop._evdata.view(-1)
        ops.rank_table(f, self._problem.senses[self._obj_index] == "max", self.weights, out=fs["aw"])
        ops.cmaes_row_weights(fs["aw"], zs, self.active, fs["w_pos"], fs["w_act"])
        ops.grad(ops.GRAD_MOMENTS, zs, fs["w_pos"], fs["zero"], fs["one"], 1.0, 1.0, out_mu=fs["local"], out_sigma=fs["scratch"])
        ops.grad(ops.GRAD_MOMENTS, ys, fs["w_pos"], fs["zero"], fs["one"], 1.0, 1.0, out_mu=fs["shaped"], out_sigma=fs["scratch"])
        ops.cmaes_vector_update(fs["local"], fs["shaped"], self.m, self.p_sigma, self.p_c, self.sigma, self._consts, self.csa_squared, fs["k"],
                                steps=self._steps_count, steps_dev=steps_dev)
        ops.weighted_syrk_update(ys, fs["w_act"], fs["k"], self.C, u=self.p_c, out=self.C)
        if steps_dev is not None or (self._steps_count + 1) % self.decompose_C_freq == 0:
            if os.environ.get("EVOTORCH_B200_EVOK_CHOLESKY", "0") == "1":
                ops.cholesky(self.C, out=self.A)  # the repo's own tile-dataflow kernel (csrc/evok_chol.cu): correct, but
                # its diagonal-tile factorisations are a serial critical path, so cuSOLVER's potrf stays the default
            else:
                torch.linalg.cholesky_ex(self.C, check_errors=False, out=(self.A, fs["info"]))

    def _step_sep_fused(self, steps_dev: Optional[torch.Tensor] = None):
        """One separable generation (cmaes.py:567-606 with diagonal C) as four kernels with no host reads.  With s = sigma * A:
        sample x_i = m + s z_i and evaluate it in one pass that also keeps q_i = ||z_i||^2 (the population is written once, or not
        at all when it is lazy) -> rank-to-weights -> the moments sum a_i z_i, sum b_i z_i^2, sum b_i over z regenerated from the
        same Philox counters (never read back) -> one update kernel for m, p_sigma, sigma, p_c, C, the stdev bounds, A and s.
        The draw takes one Philox stream id, the one the op-by-op path takes for its zs, so both paths see the same z."""
        fs = self._fused_state()
        prob, pop, n, d = self._problem, self._population, self.popsize, self._problem.solution_length
        lazy = isinstance(pop, LazySolutionBatch)
        draw = prob.next_philox_draw()
        f = pop._evdata.view(-1)
        obj = prob.evok_objective_id
        if lazy:
            # until the update below the live m and s ARE the draw's centre and stdev (what a before-eval hook or the best / worst
            # bookkeeping regenerates rows from)
            pop.recipe = draw.recipe(n, False, self.m, fs["s"])
            prob._before_eval_hook(pop)
            ops.sample_eval_sq(obj, None, self.m, fs["s"], fs["q"], n_rows=n, f=f, **draw.kwargs)
            prob._finish_evaluation(pop)
        elif obj is not None and len(prob.before_eval_hook) == 0:
            ops.sample_eval_sq(obj, pop._data, self.m, fs["s"], fs["q"], n_rows=n, f=f, **draw.kwargs)
            prob._finish_evaluation(pop)
        else:  # custom objective or before-eval hooks: sample (and keep q), then the problem's own evaluation
            ops.sample_eval_sq(ops.OBJ_NONE, pop._data, self.m, fs["s"], fs["q"], n_rows=n, **draw.kwargs)
            pop._evdata.fill_(float("nan"))
            prob.evaluate(pop)
        ops.rank_table(f, prob.senses[self._obj_index] == "max", self.weights, out=fs["aw"])
        ops.sepcma_moments(fs["aw"], fs["q"], self.active, d, local=fs["local"], S2=fs["S2"], wsum=fs["wsum"], **draw.kwargs)
        ops.sepcma_update(fs["local"], fs["S2"], fs["wsum"], self.m, self.p_sigma, self.p_c, self.sigma, self.C, self.A, fs["s"], self._consts,
                          self.csa_squared, decompose_C_freq=self.decompose_C_freq, steps=self._steps_count, steps_dev=steps_dev,
                          stdev_min=self.stdev_min, stdev_max=self.stdev_max, m_prev=fs["m_draw"], s_prev=fs["s_draw"])
        if lazy:
            # from here on the population is the one drawn from the snapshots; under a CUDA graph its recipe follows every replay
            pop.recipe = draw.between_generations().recipe(n, False, fs["m_draw"], fs["s_draw"])

    # ------------------------------------------------------------------ CUDA-graph replay of the fused generation
    def _graph_capturable(self) -> bool:
        """The fused path with a built-in objective and no evaluation hooks, and for the full covariance a Cholesky every
        generation (`decompose_C_freq == 1`; the separable update kernel schedules the decomposition from the device-side step
        counter, so it replays at any frequency)."""
        prob = self._problem
        return (self._fused_ok() and (self.separable or self.decompose_C_freq == 1) and prob.evok_objective_id is not None
                and len(prob.before_eval_hook) == 0 and len(prob.after_eval_hook) == 0 and not prob.stores_solution_stats
                and "sample_distribution" not in self.__dict__)

    def _step_graph(self):
        if self._graph is None:
            self._step_fused()  # warm every kernel / workspace / cuSOLVER handle eagerly, right before the capture
            steps_dev = torch.full((1,), self._steps_count + 1, dtype=torch.int64, device=self.m.device)
            try:
                self._graph = GenerationGraph(self._problem, lambda: self._step_fused(steps_dev), buffers=(steps_dev,))
            except Exception:  # e.g. a library call inside the step that cannot be captured on this build: stay eager
                self._use_graph = False
                torch.cuda.synchronize()
            return
        self._graph.replay()

    def __getstate__(self) -> dict:
        state = super().__getstate__()
        if state.get("_fused") is not None:
            state["_fused"] = None  # scratch buffers are rebuilt on the first step after loading
        return state

    def _step(self):
        if self._fused_ok():
            if self._use_graph and self._graph_capturable():
                self._step_graph()
            else:
                self._graph = None
                self._step_fused()
            return
        if self.separable:
            self._fused = None  # the op-by-op step replaces the state tensors: the fused buffers (and s = sigma * A) are rebuilt
        zs, ys, xs = self.sample_distribution()
        assigned_weights = self.get_population_weights(xs)
        local_m_displacement, shaped_m_displacement = self.update_m(zs, ys, assigned_weights)
        self.update_p_sigma(local_m_displacement)
        self.update_sigma()
        h_sig = self._h_sig()
        self.update_p_c(shaped_m_displacement, h_sig)
        self.update_C(zs, ys, assigned_weights, h_sig)
        if self.stdev_min is not None or self.stdev_max is not None:
            self._limit_stdev()
        if (self._steps_count + 1) % self.decompose_C_freq == 0:
            self.decompose_C()
