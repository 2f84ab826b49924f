"""Built-in vectorised objective functions with a fused evaluation kernel.

Each object is an ordinary vectorised fitness function (call it with an N x D tensor, get N fitnesses; it is marked
`__evotorch_vectorized__` like functions decorated with the reference's `@vectorized`, decorators.py:549) and
additionally carries `evok_objective_id`.  When a Problem is built around one of them, the Gaussian searchers
evaluate the population *inside* the sampling kernel (K1+K2 fused, csrc/evok_sample_eval.cu) so the N x D matrix is
written once and never re-read for evaluation.  Called directly on a CUDA fp32 population they run the stand-alone
row-reduction kernel (K2); on any other tensor the plain torch expression (same formula as the reference's README
example, README.md:86-89).

`FusedObjective` is the same for a user-defined function of sums, products, maxima and minima over the elements or over the
neighbour pairs (x_j, x_{j+1}) of a row (Rosenbrock, Griewank, Schwefel 2.21), whose element terms may also see running sums
along the row (Schwefel 1.2): its expressions are compiled at run time into the same kernels (evotorch_b200/jit.py), so every
fused path of the package takes it.
"""

from __future__ import annotations

import math
import weakref
from typing import Callable, Optional

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

    def evaluate_batched(self, values: torch.Tensor, *, seed: Optional[int] = None) -> torch.Tensor:
        """The fitnesses (..., n) of a batch of populations `values` (..., n, D), for example the asks of a batched full-covariance
        CMA-ES.  On CUDA float32 values, with a fused kernel, one launch evaluates every item: item b (in row-major order of the
        batch dimensions) draws the noise of an objective with noise from Philox key `seed` on stream b, so row i of item b gets
        the noise the batched sampler gives row i of item b with that seed (no seed: a fresh one from torch's generator).
        Anywhere else this is the torch function.  An objective with per-item data needs values of its `data_batch_shape`
        (ValueError naming both shapes otherwise)."""
        if values.ndim < 2:
            raise ValueError(f"values: expected a batch of populations of shape (..., n, D), got {tuple(values.shape)}")
        batch, (n, d) = tuple(values.shape[:-2]), tuple(values.shape[-2:])
        per_item = tuple(getattr(self, "data_batch_shape", ()))
        if per_item and per_item != batch:
            raise ValueError(f"the data of {self!r} has batch shape {per_item}, the values {batch}: every item of the data evaluates "
                             "the population of its own item")
        oid = self.evok_objective_id
        if oid is None or not ops.uses_kernels(values):
            return self._torch_fn(values)
        if hasattr(self, "compile_eval_batched"):  # a FusedObjective: its batched evaluation is compiled on the first use
            self.compile_eval_batched()
        if seed is None:
            from .algorithms.functional.misc import draw_philox_seed

            seed = draw_philox_seed()
        X = values.reshape(math.prod(batch), n, d)
        if d > 1 and X.stride(2) != 1:
            X = X.contiguous()
        return ops.evaluate_batched(oid, X, seed=seed).view(batch + (n,))

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
    sum_{j<D} term_i(x_j, j, D) or, for a term that uses xn = x_{j+1}, the pair sum sum_{j<D-1} term_i(x_j, x_{j+1}, j, D); or
    the same with a product, a maximum or a minimum in place of the sum.

        styblinski_tang = FusedObjective("styblinski_tang", sums={"s": "x**4 - 16*x**2 + 5*x"}, value="0.5 * s")
        rosenbrock = FusedObjective("rosenbrock", sums={"s": "100*(xn - x**2)**2 + (1 - x)**2"}, value="s")

    `sums` maps each sum's name to its term (an expression of x, xn, j and D), `value` is an expression of the sums and D; the
    language is described in evotorch_b200.jit.  Construction parses both (ValueError for anything outside the language),
    compiles the kernels with NVRTC for sm_90a and registers them with libevok.so; `kernel_info` holds the registers and
    spills of every kernel.  The same source compiles once per process.  A FusedObjective pickles as its expressions.

    The batched samplers of the functional API (`pgpe_ask_and_evaluate`, `cem_ask_and_evaluate`) are 8 more kernels of the same
    source, compiled on the first batched use (`compile_batched`); `batched_kernel_info` then holds their registers and spills.
    The batched evaluation (`evaluate_batched`, `cmaes_ask_and_evaluate`) is 2 more, compiled on its first use
    (`compile_eval_batched`), with `eval_batched_kernel_info`.

    `prods`, `maxs` and `mins` are reductions of terms like those of `sums`, by product, maximum and minimum; with `sums` they
    are at most 4 in all and share one namespace.  An empty reduction (a pair term at D = 1) is 0, 1, -inf or +inf, and a NaN
    term makes its product, maximum or minimum NaN (as torch.prod / amax / amin).  `running` defines at most 2 running sums
    c_j = sum_{k<=j} h(x_k, k, D), whose names the element terms of the reductions can use; `where(cond, a, b)` with one
    comparison as cond is a conditional:

        griewank = FusedObjective("griewank", sums={"s": "x**2"}, prods={"p": "cos(x / sqrt(j + 1))"}, value="1 + s / 4000 - p")
        schwefel_1_2 = FusedObjective("schwefel_1_2", running={"c": "x"}, sums={"s": "c**2"}, value="s")
        schwefel_2_21 = FusedObjective("schwefel_2_21", maxs={"m": "abs(x)"}, value="m")

    `data` gives the expressions up to 4 more names, each bound to a float32 tensor:

        lsq = FusedObjective("lsq", sums={"s": "w * (x - t)**2"}, value="s + lam * D", data={"t": t, "w": w, "lam": lam})
        shifted_rosenbrock = FusedObjective("shifted_rosenbrock", value="s", data={"o": o},
                                            sums={"s": "100*((xn - o_n) - (x - o)**2)**2 + (1 - (x - o))**2"})

    A tensor whose last dimension is 1 is a scalar (usable in the terms and in `value`); any other is a vector of the row length
    D (usable in the terms: `o` is its entry at column j, and `o_n`, in a pair term, its entry at column j + 1).  The kernels
    read the tensors themselves, which therefore must stay where they are: `obj.data["t"].copy_(new)` changes the values from
    the next generation on (also of a captured CUDA graph) without a recompile, and `with_data(**tensors)` gives a twin on
    other tensors that shares the compiled kernels, as every objective with the same expressions and kinds does.  On the kernels
    the data must be on the device of the population (ValueError).  Leading dimensions of a data tensor are batch dimensions:
    in a batched search (`pgpe_ask_and_evaluate`, `cem_ask_and_evaluate`) every item then has its own data.  All data tensors
    with batch dimensions have the same batch shape, which is the batch shape of the search (the centre and stdev are broadcast
    to it); a tensor without batch dimensions is shared by all items.  A FusedObjective with data pickles with its tensors.  In a
    multi-GPU run every rank builds its own objective: the tensors must hold the same values on every rank.

    `rand()` and `randn()` draw noise (`noisy` is then True): at most 4 occurrences in the element terms (one draw per row and
    column each) and 4 in `value` (one per row), not in pair or running terms:

        f7 = FusedObjective("f7", sums={"s": "(j + 1) * x**4"}, value="s + rand()")
        input_noise_sphere = FusedObjective("ins", sums={"s": "(x + 0.1 * randn())**2"}, value="s")

    The noise comes from the Philox key of the population's draw, so it is the same whether the population is stored or lazy,
    stepped or replayed from a CUDA graph, sharded or batched.  Rows without a draw of their own (`obj(X)`, user-set values)
    take a fresh key; on CPU tensors and other dtypes the torch function draws with torch.rand / torch.randn (the same
    distributions, not the same bits).

    `transform=(M, o)` (or `transform=M`, then o = 0) lets the terms read the transformed row y = M (x - o): `y` is its entry j
    in element and running terms, `yn` its entry j + 1 in pair terms, next to x, xn, j, D and the data:

        rot_ellipsoid = FusedObjective("rot_ellipsoid", sums={"s": "10**(6 * j / (D - 1)) * y**2"}, value="s", transform=(R, o))

    M is float32 (..., D, D), any matrix (a product Q L R is one matrix), and o float32 (..., D); their leading dimensions are
    batch dimensions under the rule of the data (one `data_batch_shape` for every batched tensor).  y_j = sum_k M[j, k] (x_k - o_k)
    with each x_k - o_k rounded first, so a row equal to o has y = 0 exactly.  M and o are bound as data are: the kernels read them
    in place, and `with_data(..., transform=(M2, o2))` swaps them.  Since a sampler produces a row one column group at a time and y
    needs the whole row, a transformed objective has no fused sampler (`evok_objective_id` is None; lazy populations raise): its
    stored populations are evaluated by its own kernels (`obj(X)`, `evaluate_batched`, and the ask-and-evaluate paths), which
    compute y in shared memory at small D and with the batched 3xTF32 GEMM above (`kernel_info` holds their registers).  The
    torch function computes y with torch.matmul after subtracting o."""

    def __init__(self, name: str, sums: Optional[dict] = None, value: Optional[str] = None, data: Optional[dict] = None, *,
                 prods: Optional[dict] = None, maxs: Optional[dict] = None, mins: Optional[dict] = None, running: Optional[dict] = None,
                 transform=None):
        from . import jit

        self.transform = _transform_pair(transform)
        spec = jit.ObjectiveSpec(sums, value, jit.data_kinds(data) if data else None, prods=prods, maxs=maxs, mins=mins,
                                 running=running, transform=self.transform is not None)
        if name in ops.OBJECTIVE_IDS and ops.OBJECTIVE_IDS[name] < ops.OBJ_USER_BASE:
            raise ValueError(f"{name!r} is the name of a built-in objective")
        self.data = dict(data) if data else {}
        self.data_batch_shape = self._data_batch_shape()
        if self.transform is not None:
            self._init_transformed(name, spec)
            return
        compiled = jit.compile_objective(spec)
        super().__init__(name, compiled.objective_id, (lambda X: spec.torch_fn(X, self.data)) if self.data else spec.torch_fn)
        self.sums, self.value, self.source = dict(spec.sums), spec.value, spec.source
        self.prods, self.maxs, self.mins, self.running = dict(spec.prods), dict(spec.maxs), dict(spec.mins), dict(spec.running)
        self.kernel_info = compiled.kernel_info
        self.batched_kernel_info = None
        self.eval_batched_kernel_info = None
        self.noisy = spec.noisy
        self._spec = spec
        if self.data:
            self._bind(compiled.objective_id)
        else:
            ops.OBJECTIVE_IDS[name] = compiled.objective_id

    def _data_batch_shape(self) -> torch.Size:
        """The one batch shape of the data and transform tensors that have batch dimensions (ValueError if they differ), () if
        none has."""
        shapes = {n: t.shape[:-1] for n, t in self.data.items() if t.ndim > 1}
        if self.transform is not None:
            M, o = self.transform
            shapes.update({k: s for k, s in (("transform M", M.shape[:-2]), ("transform o", o.shape[:-1])) if s})
        if len(set(shapes.values())) > 1:
            raise ValueError(f"data: the tensors with batch dimensions must have one batch shape, got "
                             f"{ {n: tuple(s) for n, s in shapes.items()} }")
        return next(iter(shapes.values()), torch.Size())

    def _init_transformed(self, name: str, spec) -> None:
        """The construction of an objective with a transform: its kernels are the transformed evaluation only, bound (with the
        data, if any) to `_transform_id` when every tensor is on one CUDA device; `evok_objective_id` is None."""
        from . import jit

        M, o = self.transform
        D = M.shape[-1]
        bad = [n for n, t in self.data.items() if t.shape[-1] not in (1, D)]
        if bad:
            raise ValueError(f"data[{bad[0]!r}]: a vector of length {self.data[bad[0]].shape[-1]}, the transform is {D} x {D}")
        tensors = {**self.data, "transform M": M, "transform o": o}
        if len({t.device for t in tensors.values()}) > 1:
            raise ValueError(f"the data and transform tensors are on different devices: { {n: str(t.device) for n, t in tensors.items()} }")
        compiled = jit.compile_transform(spec)
        super().__init__(name, None, lambda X: spec.torch_fn(X, self.data or None, self.transform))
        self.sums, self.value, self.source = dict(spec.sums), spec.value, spec.source
        self.prods, self.maxs, self.mins, self.running = dict(spec.prods), dict(spec.maxs), dict(spec.mins), dict(spec.running)
        self.kernel_info = compiled.kernel_info
        self.batched_kernel_info = None
        self.eval_batched_kernel_info = None
        self.noisy = spec.noisy
        self._spec = spec
        self._transform_id = None
        if M.is_cuda:
            self._transform_id = self._bind(compiled.objective_id) if self.data else compiled.objective_id

    def _bind(self, base_id: int) -> Optional[int]:
        """With the data on a CUDA device: an instance of the compiled objective bound to the tensors, which becomes this
        objective's id until the object is collected.  With the data elsewhere the objective has no fused kernel (torch_fn)."""
        from . import jit

        tensors = list(self.data.values())
        if not all(t.is_cuda for t in tensors):
            self.evok_objective_id = None
            return None
        if len({t.device for t in tensors}) > 1:
            raise ValueError(f"data: the tensors are on different devices: { {n: str(t.device) for n, t in self.data.items()} }")
        strides = []
        for n, t in self.data.items():
            # items at one stride: the batch dimensions collapse into one, and the entries of an item are contiguous
            batch = t.shape[:-1]
            flat = all(t.stride(k) == t.stride(k + 1) * t.shape[k + 1] for k in range(len(batch) - 1))
            if not (flat and (t.shape[-1] == 1 or t.stride(-1) == 1)):
                raise ValueError(f"data[{n!r}]: expected contiguous entries and batch items at one stride, got shape {tuple(t.shape)} "
                                 f"strides {t.stride()}")
            strides.append(t.stride(-2) if batch else 0)
        instance = jit.bind_instance(base_id, [t.data_ptr() for t in tensors], [t.shape[-1] for t in tensors], strides,
                                     max(math.prod(self.data_batch_shape), 1))
        ops.DATA_DEVICES[instance] = tensors[0].device
        weakref.finalize(self, _release, instance)
        if self.transform is None:
            self.evok_objective_id = instance
        return instance

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if self.transform is not None:
            return self._call_transformed(x)
        # the evaluation kernel takes one data set: per-item data, and data that is not on a CUDA device, go through torch_fn
        if self.data and (self.evok_objective_id is None or self.data_batch_shape):
            return self._torch_fn(x.unsqueeze(0))[..., 0] if x.ndim == 1 else self._torch_fn(x)
        if self.takes_key(x):  # rows without a draw of their own: a fresh key from torch's generator
            from .algorithms.functional.misc import draw_philox_seed

            return ops.evaluate_keyed(self.evok_objective_id, x, seed=draw_philox_seed(), stream_id=0)
        return super().__call__(x)

    def takes_key(self, x: torch.Tensor) -> bool:
        """True when the kernels evaluate the rows of x and the objective draws noise: then `evaluate_keyed` applies."""
        return (self.noisy and self.evok_objective_id is not None and not self.data_batch_shape and ops.uses_kernels(x) and x.ndim == 2
                and x.stride(1) == 1)

    def evaluate_keyed(self, x: torch.Tensor, draw) -> torch.Tensor:
        """The fitnesses of the rows of x (CUDA float32, `takes_key`), whose noise comes from `draw` (a `PhiloxDraw`): row i is
        global row draw.row0 + i of it, so a row the fused sampler drew with `draw` gets the fitness the sampler gave it."""
        return ops.evaluate_keyed(self.evok_objective_id, x, **draw.kwargs)

    def _call_transformed(self, x: torch.Tensor) -> torch.Tensor:
        """obj(x) with a transform: the kernels for rows (N, D) of an objective without batch dimensions and for values (..., n, D)
        whose batch shape is the objective's (or any, without batch dimensions); torch_fn for other tensors and shapes."""
        if x.ndim == 1:
            return self._torch_fn(x.unsqueeze(0))[..., 0]
        if self._transform_id is None or not ops.uses_kernels(x):
            return self._torch_fn(x)
        if x.ndim == 2:
            return self._torch_fn(x) if self.data_batch_shape else self._evaluate_transformed(x.unsqueeze(0), None)[0]
        if self.data_batch_shape and tuple(x.shape[:-2]) != tuple(self.data_batch_shape):
            return self._torch_fn(x)
        return self._evaluate_transformed(x, None)

    def evaluate_batched(self, values: torch.Tensor, *, seed: Optional[int] = None) -> torch.Tensor:
        if self.transform is None:
            return super().evaluate_batched(values, seed=seed)
        if values.ndim < 2:
            raise ValueError(f"values: expected a batch of populations of shape (..., n, D), got {tuple(values.shape)}")
        per_item = tuple(self.data_batch_shape)
        if per_item and per_item != tuple(values.shape[:-2]):
            raise ValueError(f"the data of {self!r} has batch shape {per_item}, the values {tuple(values.shape[:-2])}: every item of the "
                             "data evaluates the population of its own item")
        if self._transform_id is None or not ops.uses_kernels(values):
            return self._torch_fn(values)
        return self._evaluate_transformed(values, seed)

    evaluate_batched.__doc__ = BuiltinObjective.evaluate_batched.__doc__

    def _evaluate_transformed(self, values: torch.Tensor, seed: Optional[int]) -> torch.Tensor:
        """The transformed evaluation kernels on values (..., n, D), CUDA float32: item b of the flattened batch draws its noise
        on stream b of `seed` (None: a fresh seed from torch's generator for an objective with noise; one without takes no key)."""
        if seed is None and not self.noisy:
            seed = 0
        elif seed is None:
            from .algorithms.functional.misc import draw_philox_seed

            seed = draw_philox_seed()
        batch, (n, d) = tuple(values.shape[:-2]), tuple(values.shape[-2:])
        X = values.reshape(math.prod(batch), n, d)
        if d > 1 and X.stride(2) != 1:
            X = X.contiguous()
        M, o = self.transform
        if M.shape[-1] != d:
            raise ValueError(f"the transform of {self!r} is {M.shape[-1]} x {M.shape[-1]}, the rows have length {d}")
        # one matrix and offset per item, or one for all; the kernels read contiguous items in place
        Mi, oi = M.reshape(-1, d, d), o.reshape(-1, d)
        Mi = Mi if Mi[0].is_contiguous() else Mi.contiguous()
        oi = oi if oi[0].is_contiguous() else oi.contiguous()
        return ops.evaluate_transform_batched(self._transform_id, X, Mi, oi, seed=seed).view(batch + (n,))

    def with_data(self, transform=None, **tensors) -> "FusedObjective":
        """A twin of this objective on other tensors (all of its data names, of the same kinds): no recompile.  It keeps the
        transform, or takes `transform` (of an objective with a transform) in its place."""
        if set(tensors) != set(self.data):
            raise ValueError(f"with_data: expected the data names {list(self.data)}, got {list(tensors)}")
        if transform is not None and self.transform is None:
            raise ValueError("with_data: this objective has no transform (its terms do not read y)")
        kw = self._keywords()
        if self.transform is not None:
            kw["transform"] = self.transform if transform is None else transform
        return FusedObjective(self.name, self.sums, self.value, {n: tensors[n] for n in self.data}, **kw)

    def _keywords(self) -> dict:
        """The non-empty ones of prods, maxs, mins and running (an objective of sums only has none)."""
        return {k: v for k, v in (("prods", self.prods), ("maxs", self.maxs), ("mins", self.mins), ("running", self.running)) if v}

    def compile_batched(self) -> None:
        """Compile and attach the batched samplers (once per process for one source); fills `batched_kernel_info`."""
        _no_sampler(self)
        if self.batched_kernel_info is None:
            from . import jit

            self.batched_kernel_info = jit.compile_batched(self._spec).kernel_info

    def compile_eval_batched(self) -> None:
        """Compile and attach the batched evaluation kernels (once per process for one source); fills `eval_batched_kernel_info`."""
        _no_sampler(self)
        if self.eval_batched_kernel_info is None:
            from . import jit

            self.eval_batched_kernel_info = jit.compile_eval_batched(self._spec).kernel_info

    def __reduce__(self):
        args = (self.name, self.sums, self.value) + ((self.data,) if self.data else ())
        kw = self._keywords()
        if self.transform is not None:
            kw["transform"] = self.transform
        if not kw:
            return (FusedObjective, args)
        return (_make_fused, (args, kw))

    def __repr__(self) -> str:
        data = ", data={" + ", ".join(f"{n!r}: {tuple(t.shape)}" for n, t in self.data.items()) + "}" if self.data else ""
        more = "".join(f", {k}={v!r}" for k, v in self._keywords().items())
        if self.transform is not None:
            more += f", transform=(M {tuple(self.transform[0].shape)}, o {tuple(self.transform[1].shape)})"
        return f"FusedObjective({self.name!r}, sums={self.sums!r}, value={self.value!r}{data}{more})"


def _make_fused(args: tuple, keywords: dict) -> FusedObjective:
    """Unpickle a FusedObjective with keyword reductions, running sums or a transform."""
    return FusedObjective(*args, **keywords)


def _transform_pair(transform) -> Optional[tuple]:
    """(M, o) of the `transform` argument: a pair, or M alone (o = 0); None for none.  ValueError for a matrix that is not square,
    an offset of another length, or tensors that are not float32."""
    if transform is None:
        return None
    M, o = transform if isinstance(transform, (tuple, list)) and len(transform) == 2 else (transform, None)
    if not (isinstance(M, torch.Tensor) and M.dtype == torch.float32 and M.ndim >= 2 and M.shape[-1] == M.shape[-2] >= 1):
        what = f"{tuple(M.shape)} {M.dtype}" if isinstance(M, torch.Tensor) else type(M).__name__
        raise ValueError(f"transform: M must be a square float32 matrix (..., D, D), got {what}")
    D = M.shape[-1]
    if o is None:
        o = torch.zeros(D, dtype=torch.float32, device=M.device)
    if not (isinstance(o, torch.Tensor) and o.dtype == torch.float32 and o.ndim >= 1 and o.shape[-1] == D):
        what = f"{tuple(o.shape)} {o.dtype}" if isinstance(o, torch.Tensor) else type(o).__name__
        raise ValueError(f"transform: o must be a float32 vector (..., D) with D = {D} (M is {D} x {D}), got {what}")
    if o.device != M.device:
        raise ValueError(f"transform: M is on {M.device}, o on {o.device}")
    return (M, o)


def is_transformed(objective) -> bool:
    """True for a FusedObjective with a transform (whose terms read y = M (x - o)): it has no fused sampler and is evaluated on
    stored populations by its own kernels."""
    return isinstance(objective, FusedObjective) and objective.transform is not None


def _no_sampler(obj: FusedObjective) -> None:
    if obj.transform is not None:
        raise ValueError(f"{obj!r} reads the transformed row y = M (x - o), which no sampler produces (it samples one column group "
                         "at a time): it is evaluated on stored populations only")


def _release(instance_id: int) -> None:
    from . import jit

    ops.DATA_DEVICES.pop(instance_id, None)
    jit.release_instance(instance_id)


sphere = BuiltinObjective("sphere", ops.OBJ_SPHERE, _sphere)
rastrigin = BuiltinObjective("rastrigin", ops.OBJ_RASTRIGIN, _rastrigin)
ackley = BuiltinObjective("ackley", ops.OBJ_ACKLEY, _ackley)

__all__ = ["sphere", "rastrigin", "ackley", "BuiltinObjective", "FusedObjective"]
