"""Search distributions (mirrors evotorch.distributions of the reference, distributions.py:40-1016).

The public surface is the reference's: `sample(num_solutions=None, *, out=None, generator=None)`,
`compute_gradients(samples, fitnesses, *, objective_sense, ranking_method=None) -> dict`,
`update_parameters(gradients, *, learning_rates=None, optimizers=None) -> Distribution`, `modified_copy`, `to`.
What differs is what runs underneath for CUDA float32 tensors:

  sample             -> K1  fused Philox4x32-10 -> Box-Muller -> mu +/- sigma*z write   (csrc/evok_sample_eval.cu)
  compute_gradients  -> K3  radix-sort ranking + K4 one fused weighted column reduction (csrc/evok_rank.cu, evok_grad.cu)
  update_parameters  -> K5  single-launch ClipUp/Adam step and sigma update             (csrc/evok_update.cu)

CPU tensors (BASELINE config 1, the gloo tests) and non-fp32 dtypes use the generic torch implementation in this
file.  A CUDA fp32 tensor never reaches the torch implementation: if libevok.so is missing the call raises.
"""

from __future__ import annotations

import math
from copy import copy
from typing import Any, Iterable, Optional

import torch

from . import ops
from .core import PhiloxRecipe, PhiloxSamples
from .tools.cloning import Clonable
from .tools.readonlytensor import as_plain_tensor
from .tools.misc import extract_generator, make_gaussian, to_torch_dtype
from .tools.ranking import rank


def _philox_source(generator: Any):
    """Objects that hand out Philox draws (our Problem with rng="philox") select the K1 sampler; a bare torch.Generator (or
    None) selects torch's own RNG."""
    return generator if (generator is not None and hasattr(generator, "next_philox_draw")
                         and getattr(generator, "rng", "philox") == "philox") else None


class Distribution(Clonable):
    """Base class of all search distributions (distributions.py:40-410)."""

    MANDATORY_PARAMETERS: set = set()
    OPTIONAL_PARAMETERS: set = set()
    PARAMETER_NDIMS: dict = {}

    def __init__(self, *, solution_length: int, parameters: dict, dtype=None, device=None):
        self.__solution_length = int(solution_length)
        found = 0
        for name in parameters:
            if name in self.MANDATORY_PARAMETERS:
                found += 1
            elif name not in self.OPTIONAL_PARAMETERS:
                raise ValueError(f"Unrecognized parameter: {name!r}")
        if found < len(self.MANDATORY_PARAMETERS):
            raise ValueError(
                f"Not all mandatory parameters of this Distribution were specified. Mandatory parameters of this distribution:"
                f" {self.MANDATORY_PARAMETERS}; optional parameters of this distribution: {self.OPTIONAL_PARAMETERS};"
                f" encountered parameters: {set(parameters.keys())}."
            )
        tensors = [v for v in parameters.values() if isinstance(v, torch.Tensor)]
        self.__dtype = to_torch_dtype(dtype) if dtype is not None else tensors[0].dtype
        self.__device = torch.device(device) if device is not None else tensors[0].device
        self.__parameters = {
            k: (v.to(dtype=self.__dtype, device=self.__device) if isinstance(v, torch.Tensor) else v) for k, v in parameters.items()
        }

    # ------------------------------------------------------------------ plumbing
    @property
    def solution_length(self) -> int:
        return self.__solution_length

    @property
    def device(self) -> torch.device:
        return self.__device

    @property
    def dtype(self) -> torch.dtype:
        return self.__dtype

    @property
    def parameters(self) -> dict:
        return self.__parameters

    def to(self, device) -> "Distribution":
        if torch.device(self.device) == torch.device(device):
            return self
        device = torch.device(device)
        if device.type == "cuda":
            # host-resident distribution driving a CUDA problem (core.py:2958 `dist_on_cpu` protocol in reverse): parameters that
            # live in pinned memory are copied asynchronously on the current stream (the kernels that consume them are ordered
            # behind the copies), so the transfer costs no host synchronisation
            params = {k: (v.to(device, non_blocking=v.is_pinned()) if isinstance(v, torch.Tensor) else v) for k, v in self.parameters.items()}
            return type(self)(solution_length=self.solution_length, parameters=params, device=device)
        return type(self)(solution_length=self.solution_length, parameters=self.parameters, device=device)

    def modified_copy(self, *, dtype=None, device=None, **parameters) -> "Distribution":
        new_parameters = copy(self.parameters)
        new_parameters.update(parameters)
        return type(self)(parameters=new_parameters, dtype=self.dtype if dtype is None else dtype,
                          device=self.device if device is None else device)

    def make_empty(self, *, num_solutions: int) -> torch.Tensor:
        return torch.empty(int(num_solutions), self.solution_length, dtype=self.dtype, device=self.device)

    def make_zeros(self, *, num_solutions: int) -> torch.Tensor:
        return torch.zeros(int(num_solutions), self.solution_length, dtype=self.dtype, device=self.device)

    # ------------------------------------------------------------------ sampling
    def _fill(self, out: torch.Tensor, *, generator: Any = None):
        raise NotImplementedError

    def sample(self, num_solutions: Optional[int] = None, *, out: Optional[torch.Tensor] = None, generator: Any = None) -> torch.Tensor:
        """Fill `out` (N x solution_length) in place, or allocate num_solutions rows (distributions.py:155-216)."""
        if (num_solutions is not None) and (out is not None):
            raise ValueError("Received both `num_solutions` and `out` with values other than None. Please provide only one of them.")
        if (num_solutions is None) and (out is None):
            raise ValueError("Received both `num_solutions` and `out` as None. Please provide one of these arguments.")
        if out is None:
            out = self.make_empty(num_solutions=int(num_solutions))
        else:
            if out.ndim != 2:
                raise ValueError(f"The `sample(...)` method can fill only 2-dimensional tensors. However, the provided `out` tensor has"
                                 f" {out.ndim} dimensions, its shape being {out.shape}.")
            if out.shape[1] != self.solution_length:
                raise ValueError(f"The solution length declared by this distribution is {self.solution_length}. However, the provided"
                                 f" `out` tensor has {out.shape[1]} columns.")
        self._fill(out, generator=generator)
        return out

    # ------------------------------------------------------------------ gradients
    def _compute_gradients(self, samples: torch.Tensor, weights: torch.Tensor, ranking_used: Optional[str]) -> dict:
        raise NotImplementedError

    def compute_gradients(self, samples: torch.Tensor, fitnesses: torch.Tensor, *, objective_sense: str,
                          ranking_method: Optional[str] = None) -> dict:
        """Rank the fitnesses and reduce the utility-weighted gradients (distributions.py:236-299)."""
        if objective_sense == "max":
            higher_is_better = True
        elif objective_sense == "min":
            higher_is_better = False
        else:
            raise ValueError(f'`objective_sense` was expected as "min" or as "max". However, it was encountered as {objective_sense!r}.')
        if ranking_method is None:
            ranking_method = "raw"
        fitnesses = as_plain_tensor(torch.as_tensor(fitnesses, dtype=self.dtype))  # e.g. `batch.evals[:, 0]` is a ReadOnlyTensor
        samples = as_plain_tensor(samples)
        [num_samples, _] = samples.shape
        [num_fitnesses] = fitnesses.shape
        if num_samples != num_fitnesses:
            raise ValueError(f"The number of samples and the number of fitnesses do not match: {num_samples} != {num_fitnesses}.")
        weights = rank(fitnesses, ranking_method=ranking_method, higher_is_better=higher_is_better)
        return self._compute_gradients(samples, weights, ranking_method)

    def update_parameters(self, gradients: dict, *, learning_rates: Optional[dict] = None, optimizers: Optional[dict] = None) -> "Distribution":
        raise NotImplementedError

    def _follow_gradient(self, param_name: str, x: torch.Tensor, *, learning_rates: Optional[dict] = None,
                         optimizers: Optional[dict] = None) -> torch.Tensor:
        """lr * g, optimizer.ascent(g), or g itself (distributions.py:372-392)."""
        x = torch.as_tensor(x, dtype=self.dtype, device=self.device)
        lr = (learning_rates or {}).get(param_name)
        opt = (optimizers or {}).get(param_name)
        if lr is None and opt is None:
            return x
        if opt is None:
            return lr * x
        if lr is None:
            return opt.ascent(x)
        raise ValueError("Encountered both `learning_rate` and `optimizer` as values other than None.")


def _weighted_colsum(w: torch.Tensor, m: torch.Tensor) -> torch.Tensor:
    """sum_i w_i * m_i over rows (generic torch path; the reference spells this total(dot(w, m)), tools/misc.py:1089-1110)."""
    return torch.mv(m.T, w) if m.dtype.is_floating_point else torch.sum(w.unsqueeze(-1) * m, dim=0)


class SeparableGaussian(Distribution):
    """Separable Gaussian N(mu, diag(sigma^2)) of PGPE (non-symmetric) and CEM (distributions.py:413-613)."""

    MANDATORY_PARAMETERS = {"mu", "sigma"}
    OPTIONAL_PARAMETERS = {"divide_mu_grad_by", "divide_sigma_grad_by", "parenthood_ratio"}
    PARAMETER_NDIMS = {"mu": 1, "sigma": 1}
    SYMMETRIC = False
    GRAD_FORM = ops.GRAD_SEPARABLE

    def __init__(self, parameters: dict, *, solution_length: Optional[int] = None, device=None, dtype=None):
        [mu_length] = parameters["mu"].shape
        [sigma_length] = parameters["sigma"].shape
        if solution_length is None:
            solution_length = mu_length
        elif solution_length != mu_length:
            raise ValueError(f"The argument `solution_length` does not match the length of `mu` provided in `parameters`."
                             f" solution_length={solution_length}, parameters[\"mu\"]={mu_length}.")
        if mu_length != sigma_length:
            raise ValueError(f"The tensors `mu` and `sigma` provided within `parameters` have mismatching lengths."
                             f" parameters[\"mu\"]={mu_length}, parameters[\"sigma\"]={sigma_length}.")
        super().__init__(solution_length=solution_length, parameters=parameters, device=device, dtype=dtype)

    @property
    def mu(self) -> torch.Tensor:
        return self.parameters["mu"]

    @mu.setter
    def mu(self, new_mu: Iterable):
        self.parameters["mu"] = torch.as_tensor(new_mu, dtype=self.dtype, device=self.device)

    @property
    def sigma(self) -> torch.Tensor:
        return self.parameters["sigma"]

    @sigma.setter
    def sigma(self, new_sigma: Iterable):
        self.parameters["sigma"] = torch.as_tensor(new_sigma, dtype=self.dtype, device=self.device)

    # -------------------------------------------------- sampling (K1)
    def _fill(self, out: torch.Tensor, *, generator: Any = None):
        src = _philox_source(generator)
        if src is not None and ops.uses_kernels(out) and out.stride(1) == 1:
            if self.SYMMETRIC and out.shape[0] % 2 != 0:
                raise ValueError(f"Symmetric sampling cannot be done if the leftmost dimension of the target tensor is odd: {tuple(out.shape)}")
            ops.sample_eval(ops.OBJ_NONE, out, self.mu.contiguous(), self.sigma.contiguous(), n_rows=out.shape[0],
                            symmetric=self.SYMMETRIC, **src.next_philox_draw().kwargs)
        else:
            make_gaussian(out=out, center=self.mu, stdev=self.sigma, symmetric=self.SYMMETRIC, generator=extract_generator(generator))

    # -------------------------------------------------- gradients (K4)
    def _grad_scale(self, param_name: str, weights: torch.Tensor, n_total: Optional[int] = None):
        """divide_*_grad_by -> (host scale, optional device divisor) (distributions.py:517-536).  `n_total`: the population
        size when `weights` is only a shard's slice."""
        option = self.parameters.get(f"divide_{param_name}_grad_by")
        n = weights.shape[0] if n_total is None else int(n_total)
        if option is None:
            return 1.0, None
        if option == "num_solutions":
            return 1.0 / n, None
        if option == "num_directions":
            return 1.0 / (n // 2), None
        if option == "total_weight":
            return 1.0, torch.sum(torch.abs(weights))
        if option == "weight_stdev":
            return 1.0, torch.std(weights)
        raise ValueError(f"The parameter divide_{param_name}_grad_by has an unrecognized value: {option}")

    def _prepared_weights(self, weights: torch.Tensor, ranking_used: Optional[str]) -> torch.Tensor:
        """`w - mean(w)` unless the ranking is already zero-centred (distributions.py:562-563, :722-723)."""
        if ranking_used not in self._UNTOUCHED_RANKINGS:
            if ops.uses_kernels(weights):
                return ops.weights_adjust_(weights.clone(), 1)
            return weights - torch.mean(weights)
        return weights

    _UNTOUCHED_RANKINGS = ("centered", "normalized")  # utilities that `_prepared_weights` passes through unchanged

    def _weighted_sums(self, form: int, samples, w: torch.Tensor, scale_mu: float, scale_sigma: float, peer=None) -> tuple:
        """(scale_mu * sum_r a_r eps_r, scale_sigma * sum_r b_r g(eps_r)) -- the K4 kernel, or its torch restatement.
        `samples` is a values tensor, a `PhiloxRecipe` (lazy population: every row is regenerated) or a `PhiloxSamples` (values
        the fused sampler wrote from mu / sigma, untouched since: part of the rows is rebuilt).  `peer`: a sharded generation
        over NVLink peer memory, where the kernel pushes this shard's sums to every GPU and the result is the global sums."""
        if isinstance(samples, PhiloxSamples):
            values, recipe = samples.values, samples.recipe
        elif isinstance(samples, PhiloxRecipe):
            values, recipe = None, samples
        else:
            values, recipe = samples, None
        w, mu, sigma = w.contiguous(), self.mu.contiguous(), self.sigma.contiguous()
        if peer is not None:  # reads the values where there are any, regenerates them otherwise
            ops.grad_push(form, values, w, mu, sigma, scale_mu=scale_mu, scale_sigma=scale_sigma, peer=peer,
                          **(recipe.draw.kwargs if values is None else {}))
            return peer.reduce_gradients()
        if values is None:
            return ops.grad_regen(form, w, mu, sigma, scale_mu=scale_mu, scale_sigma=scale_sigma, **recipe.draw.kwargs)
        if recipe is not None and ops.uses_kernels(w):
            return ops.grad_hybrid(form, values, w, mu, sigma, scale_mu=scale_mu, scale_sigma=scale_sigma, **recipe.draw.kwargs)
        if ops.uses_kernels(values) and ops.uses_kernels(w):
            return ops.grad(form, values, w, mu, sigma, scale_mu, scale_sigma)
        if form == ops.GRAD_SYMMETRIC:
            eps = values[0::2] - mu
            a, b = (w[0::2] - w[1::2]) / 2, (w[0::2] + w[1::2]) / 2
        else:
            eps = values - mu
            a = b = w
        if form == ops.GRAD_EXP:
            g = ((eps / sigma) ** 2) - 1
        elif form == ops.GRAD_MOMENTS:
            g = eps**2
        else:
            g = ((eps**2) - (sigma**2)) / sigma
        return _weighted_colsum(a, eps) * scale_mu, _weighted_colsum(b, g) * scale_sigma

    def accepts_local_weights(self, ranking_used: Optional[str]) -> bool:
        """True when a shard's gradient contribution needs nothing but the utilities of its OWN rows (no statistic of the whole
        utility vector: no mean subtraction, no sum / stdev divisor, no elite selection) -- the condition for the sharded
        ranking, where no GPU ever holds the full utility vector."""
        if "parenthood_ratio" in self.parameters:
            return False
        for name in ("mu", "sigma"):
            if self.parameters.get(f"divide_{name}_grad_by") not in (None, "num_solutions", "num_directions"):
                return False
        return ranking_used in self._UNTOUCHED_RANKINGS and ranking_used in ("centered", "linear", "nes")

    def partial_gradients(self, samples: torch.Tensor, all_weights: torch.Tensor, row0: int, ranking_used: Optional[str],
                          local_weights_of: Optional[int] = None, peer=None) -> dict:
        """Gradient contribution of a row shard.  `samples` are rows [row0, row0 + n) of a population whose utilities are
        `all_weights` (ranked over the WHOLE population).  The dictionaries of all shards add up (all-reduce) to what
        `finalize_gradients` turns into the result of `compute_gradients` on the whole population.
        `local_weights_of=N`: `all_weights` holds only the utilities of THIS shard's rows, of a population of N solutions
        (sharded ranking; see `accepts_local_weights`).  With `peer` (an evotorch_b200.peer.PeerExchange) the kernels do the
        all-reduce: the result is already summed over the ranks."""
        n_local = samples.shape[0]
        if local_weights_of is not None:
            if not self.accepts_local_weights(ranking_used):
                raise ValueError("this distribution / ranking needs the utilities of the whole population")
            smu, _ = self._grad_scale("mu", all_weights, local_weights_of)
            ssig, _ = self._grad_scale("sigma", all_weights, local_weights_of)
            gmu, gsig = self._weighted_sums(self.GRAD_FORM, samples, all_weights, smu, ssig, peer)
            return {"mu": gmu, "sigma": gsig}
        if "parenthood_ratio" in self.parameters:  # CEM elite moments (distributions.py:538-546)
            num_elites = math.floor(all_weights.shape[0] * self.parameters["parenthood_ratio"])
            if ops.uses_kernels(all_weights):
                mask = ops.elite_mask(all_weights.contiguous(), num_elites)
            else:
                mask = torch.zeros_like(all_weights)
                mask[torch.argsort(all_weights, descending=True, stable=True)[:num_elites]] = 1
            s1, s2 = self._weighted_sums(ops.GRAD_MOMENTS, samples, mask[row0:row0 + n_local], 1.0, 1.0, peer)
            return {"elite_sum": s1, "elite_sqsum": s2}
        w = self._prepared_weights(all_weights, ranking_used)
        smu, dmu = self._grad_scale("mu", w)
        ssig, dsig = self._grad_scale("sigma", w)
        gmu, gsig = self._weighted_sums(self.GRAD_FORM, samples, w[row0:row0 + n_local], smu, ssig, peer)
        if dmu is not None:
            gmu = gmu / dmu
        if dsig is not None:
            gsig = gsig / dsig
        return {"mu": gmu, "sigma": gsig}

    def finalize_gradients(self, summed: dict, num_solutions: int) -> dict:
        if "elite_sum" in summed:
            num_elites = math.floor(num_solutions * self.parameters["parenthood_ratio"])
            s1, s2 = summed["elite_sum"], summed["elite_sqsum"]
            if ops.uses_kernels(s1):
                gmu, gsig = ops.cem_finalize(s1.contiguous(), s2.contiguous(), self.sigma.contiguous(), num_elites)
            else:
                gmu = s1 / num_elites
                var = (s2 - s1 * s1 / num_elites) / (num_elites - 1)
                gsig = torch.sqrt(torch.clamp_min(var, 0)) - self.sigma
            return {"mu": gmu, "sigma": gsig}
        return summed

    def _compute_gradients(self, samples: torch.Tensor, weights: torch.Tensor, ranking_used: Optional[str]) -> dict:
        return self.finalize_gradients(self.partial_gradients(samples, weights, 0, ranking_used), weights.shape[0])

    # -------------------------------------------------- update (K5)
    def update_parameters(self, gradients: dict, *, learning_rates: Optional[dict] = None, optimizers: Optional[dict] = None):
        """mu + follow(grad_mu), sigma + follow(grad_sigma) -> a NEW distribution (distributions.py:581-596)."""
        new_mu = self.mu + self._follow_gradient("mu", gradients["mu"], learning_rates=learning_rates, optimizers=optimizers)
        new_sigma = self.sigma + self._follow_gradient("sigma", gradients["sigma"], learning_rates=learning_rates, optimizers=optimizers)
        return self.modified_copy(mu=new_mu, sigma=new_sigma)

    def relative_entropy(dist_0: "SeparableGaussian", dist_1: "SeparableGaussian") -> float:
        """KL(dist_0 || dist_1) of two separable Gaussians (distributions.py:598-613)."""
        cov_0, cov_1 = dist_0.sigma.pow(2.0), dist_1.sigma.pow(2.0)
        mu_delta = dist_1.mu - dist_0.mu
        k = dist_0.solution_length
        return 0.5 * (torch.sum(cov_0 / cov_1) - k + torch.sum(mu_delta.pow(2.0) / cov_1) + torch.sum(torch.log(cov_1))
                      - torch.sum(torch.log(cov_0)))


class SymmetricSeparableGaussian(SeparableGaussian):
    """Antithetic separable Gaussian of PGPE: rows 2k / 2k+1 are mu + sigma*z_k and mu - sigma*z_k
    (distributions.py:616-773)."""

    SYMMETRIC = True
    GRAD_FORM = ops.GRAD_SYMMETRIC


class ExpSeparableGaussian(SeparableGaussian):
    """Separable Gaussian with exponential sigma update, as used by SNES (distributions.py:776-810)."""

    OPTIONAL_PARAMETERS: set = set()
    GRAD_FORM = ops.GRAD_EXP

    def _prepared_weights(self, weights: torch.Tensor, ranking_used: Optional[str]) -> torch.Tensor:
        """`w / sum|w|` unless the utilities are NES utilities (distributions.py:784-785)."""
        if ranking_used != "nes":
            if ops.uses_kernels(weights):
                return ops.weights_adjust_(weights.clone(), 2)
            return weights / torch.sum(torch.abs(weights))
        return weights

    _UNTOUCHED_RANKINGS = ("nes",)

    def update_parameters(self, gradients: dict, *, learning_rates: Optional[dict] = None, optimizers: Optional[dict] = None):
        """mu + follow(grad_mu); sigma * exp(0.5 * follow(grad_sigma)) (distributions.py:795-810)."""
        new_mu = self.mu + self._follow_gradient("mu", gradients["mu"], learning_rates=learning_rates, optimizers=optimizers)
        new_sigma = self.sigma * torch.exp(
            0.5 * self._follow_gradient("sigma", gradients["sigma"], learning_rates=learning_rates, optimizers=optimizers))
        return self.modified_copy(mu=new_mu, sigma=new_sigma)


class ExpGaussian(Distribution):
    """Full-covariance Gaussian N(mu, A^T A) with exponential-map update, as used by XNES (distributions.py:813-1016).
    The contractions are dense D x D products: they go to the GEMM library (cuBLAS through torch.matmul); the N x D x D
    temporary the reference materialises at :980-984 is replaced by Z^T diag(w) Z."""

    MANDATORY_PARAMETERS = {"mu", "sigma"}
    OPTIONAL_PARAMETERS = {"sigma_inv"}
    PARAMETER_NDIMS = {"mu": 1, "sigma": 2, "sigma_inv": 2}

    def __init__(self, parameters: dict, *, solution_length: Optional[int] = None, device=None, dtype=None):
        parameters = dict(parameters)
        [mu_length] = parameters["mu"].shape
        if parameters["sigma"].ndim == 1:
            parameters["sigma"] = torch.diag(parameters["sigma"])
        if "sigma_inv" not in parameters:
            parameters["sigma_inv"] = torch.inverse(parameters["sigma"])
        [sigma_length, _] = parameters["sigma"].shape
        if solution_length is None:
            solution_length = mu_length
        elif solution_length != mu_length:
            raise ValueError(f"The argument `solution_length` does not match the length of `mu` provided in `parameters`.")
        if mu_length != sigma_length:
            raise ValueError("The tensors `mu` and `sigma` provided within `parameters` have mismatching lengths.")
        super().__init__(solution_length=solution_length, parameters=parameters, device=device, dtype=dtype)
        self.eye = torch.eye(solution_length, dtype=self.dtype, device=self.device)

    @property
    def mu(self) -> torch.Tensor:
        return self.parameters["mu"]

    @property
    def sigma(self) -> torch.Tensor:
        return self.parameters["sigma"]

    @property
    def sigma_inv(self) -> torch.Tensor:
        return self.parameters["sigma_inv"]

    A = sigma
    A_inv = sigma_inv

    @property
    def cov(self) -> torch.Tensor:
        return self.sigma.transpose(0, 1) @ self.sigma

    def to_global_coordinates(self, local_coordinates: torch.Tensor) -> torch.Tensor:
        """mu + z A^T (distributions.py:928-938); the tensor-core GEMM with the `+ mu` epilogue on CUDA fp32."""
        if ops.uses_kernels(local_coordinates) and ops.uses_kernels(self.A) and local_coordinates.ndim == 2:
            z = local_coordinates.contiguous()
            out = torch.empty_like(z)
            ops.gemm_nt(z, self.A.contiguous(), torch.empty_like(z), out2=out, bias=self.mu.contiguous())
            return out
        return self.mu.unsqueeze(0) + (self.A @ local_coordinates.T).T

    def to_local_coordinates(self, global_coordinates: torch.Tensor) -> torch.Tensor:
        """(x - mu) A^-T (distributions.py:940-950)."""
        centered = global_coordinates - self.mu.unsqueeze(0)
        if ops.uses_kernels(centered) and ops.uses_kernels(self.A_inv) and centered.ndim == 2:
            return ops.gemm_nt(centered.contiguous(), self.A_inv.contiguous())
        return (self.A_inv @ centered.T).T

    def _fill(self, out: torch.Tensor, *, generator: Any = None):
        make_gaussian(out=out, generator=extract_generator(generator))
        out[:] = self.to_global_coordinates(out)

    def _compute_gradients(self, samples: torch.Tensor, weights: torch.Tensor, ranking_used: Optional[str]) -> dict:
        z = self.to_local_coordinates(samples)
        if ranking_used not in ("centered", "normalized"):
            weights = weights - torch.mean(weights)
        d_grad = torch.mv(z.T, weights)
        if ops.uses_kernels(z) and ops.uses_kernels(weights):
            zc = z.contiguous()
            outer = ops.gemm_nt(ops.transpose_scale(zc, weights.contiguous()), ops.transpose_scale(zc))  # Z^T diag(w) Z
        else:
            outer = (z.T * weights) @ z
        m_grad = outer - torch.sum(weights) * self.eye
        return {"d": d_grad, "M": m_grad}

    def update_parameters(self, gradients: dict, *, learning_rates: Optional[dict] = None, optimizers: Optional[dict] = None):
        learning_rates = dict(learning_rates or {})
        learning_rates.setdefault("d", learning_rates.get("mu"))
        learning_rates.setdefault("M", learning_rates.get("sigma"))
        optimizers = dict(optimizers or {})
        if "mu" in optimizers:  # the searcher registers its optimizer under "mu"; XNES follows "d" with it
            optimizers.setdefault("d", optimizers["mu"])
            learning_rates["d"] = None
        update_d = self._follow_gradient("d", gradients["d"], learning_rates=learning_rates, optimizers=optimizers)
        update_m = self._follow_gradient("M", gradients["M"], learning_rates=learning_rates, optimizers=optimizers)
        new_mu = self.mu + torch.mv(self.A, update_d)
        new_a = self.A @ torch.matrix_exp(0.5 * update_m)
        new_a_inv = torch.matrix_exp(-0.5 * update_m) @ self.A_inv
        return self.modified_copy(mu=new_mu, sigma=new_a, sigma_inv=new_a_inv)
