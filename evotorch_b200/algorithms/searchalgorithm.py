"""Driver loop, hooks and lazily computed status of all search algorithms (mirrors
evotorch.algorithms.searchalgorithm, searchalgorithm.py:34-584).  Pure host-side bookkeeping; status values are
only computed when something (a logger, the user) reads them, so reading nothing costs no device synchronisation."""

from __future__ import annotations

import io
import os
from collections.abc import Mapping
from datetime import datetime
from typing import Any, Iterable, Optional

import torch

from ..core import Hook, Problem, SolutionBatch


class LazyReporter:
    """Status dictionary whose entries are produced on first access per generation (searchalgorithm.py:34-182)."""

    @staticmethod
    def _missing_status_producer():
        return None

    def __init__(self, **kwargs):
        self.__getters = kwargs
        self.__computed = {}

    def get_status_value(self, key: Any) -> Any:
        if key not in self.__computed:
            self.__computed[key] = self.__getters[key]()
        return self.__computed[key]

    def has_status_key(self, key: Any) -> bool:
        return key in self.__getters

    def iter_status_keys(self):
        return self.__getters.keys()

    def clear_status(self):
        self.__computed.clear()

    def is_status_computed(self, key) -> bool:
        return key in self.__computed

    def update_status(self, additional_status: Mapping):
        for k, v in additional_status.items():
            if k not in self.__getters:
                self.__getters[k] = LazyReporter._missing_status_producer
            self.__computed[k] = v

    def add_status_getters(self, getters: Mapping):
        self.__getters.update(getters)

    @property
    def status(self) -> "LazyStatusDict":
        return LazyStatusDict(self)


class LazyStatusDict(Mapping):
    def __init__(self, lazy_reporter: LazyReporter):
        super().__init__()
        self.__lazy_reporter = lazy_reporter

    def __getitem__(self, key: Any) -> Any:
        return self.__lazy_reporter.get_status_value(key)

    def __len__(self) -> int:
        return len(list(self.__lazy_reporter.iter_status_keys()))

    def __iter__(self):
        yield from self.__lazy_reporter.iter_status_keys()

    def __contains__(self, key: Any) -> bool:
        return self.__lazy_reporter.has_status_key(key)

    def _to_string(self) -> str:
        with io.StringIO() as f:
            print("<" + type(self).__name__, file=f)
            for k in self.__lazy_reporter.iter_status_keys():
                r = repr(self.__lazy_reporter.get_status_value(k)) if self.__lazy_reporter.is_status_computed(k) else "<not yet computed>"
                print("   ", k, "=", r, file=f)
            print(">", end="", file=f)
            return f.getvalue()

    __str__ = __repr__ = _to_string


class SearchAlgorithm(LazyReporter):
    """Base class: `step()` runs one generation (`_step`) between the hooks, `run(n)` repeats it (searchalgorithm.py:240-447)."""

    def __init__(self, problem: Problem, **kwargs):
        super().__init__(**kwargs)
        self._problem = problem
        self._before_step_hook = Hook()
        self._after_step_hook = Hook()
        self._log_hook = Hook()
        self._end_of_run_hook = Hook()
        self._steps_count: int = 0
        self._first_step_datetime: Optional[datetime] = None

    @property
    def problem(self) -> Problem:
        return self._problem

    @property
    def before_step_hook(self) -> Hook:
        return self._before_step_hook

    @property
    def after_step_hook(self) -> Hook:
        return self._after_step_hook

    @property
    def log_hook(self) -> Hook:
        return self._log_hook

    @property
    def end_of_run_hook(self) -> Hook:
        return self._end_of_run_hook

    @property
    def step_count(self) -> int:
        return self._steps_count

    steps_count = step_count

    def step(self):
        self._before_step_hook()
        self.clear_status()
        if self._first_step_datetime is None:
            self._first_step_datetime = datetime.now()
        self._step()
        self._steps_count += 1
        self.update_status({"iter": self._steps_count})
        self.update_status(self._problem.status)
        self.update_status(self._after_step_hook.accumulate_dict())
        if len(self._log_hook) >= 1:
            self._log_hook(dict(self.status))

    def _step(self):
        raise NotImplementedError

    def run(self, num_generations: int, *, reset_first_step_datetime: bool = True):
        if reset_first_step_datetime:
            self.reset_first_step_datetime()
        for _ in range(int(num_generations)):
            self.step()
        if len(self._end_of_run_hook) >= 1:
            self._end_of_run_hook(dict(self.status))

    @property
    def first_step_datetime(self) -> Optional[datetime]:
        return self._first_step_datetime

    def reset_first_step_datetime(self):
        self._first_step_datetime = None

    @property
    def is_terminated(self) -> bool:
        return False


class CUDAGraphMixin:
    """`enable_cuda_graph()` for the searchers that can replay a whole generation from one CUDA graph (`.cudagraph`).
    `_graph` is the captured `GenerationGraph` or None; each searcher's `_graph_capturable()` says when it may be used."""

    def __init__(self):
        self._use_graph = os.environ.get("EVOTORCH_B200_CUDA_GRAPH", "0") == "1"
        self._graph = None

    def enable_cuda_graph(self, enabled: bool = True):
        """Capture one generation into a CUDA graph and replay it from `step()`: one graph launch per generation instead of
        the kernel launches and their Python glue.  The trajectory is bit-identical to eager stepping: the sampler reads a
        device-side generation counter that an in-graph kernel increments.  Stepping stays eager while the configuration is
        not capturable (hooks, non-fused paths, ...); calling this again drops the captured graph."""
        self._use_graph = bool(enabled)
        self._graph = None
        return self

    def __getstate__(self) -> dict:
        """Everything but the captured CUDA graph (re-captured on the first step after loading)."""
        state = dict(self.__dict__)
        state["_graph"] = None
        return state


class SinglePopulationAlgorithmMixin:
    """Adds pop_best / pop_best_eval / mean_eval / median_eval status entries for algorithms with a `population`
    (searchalgorithm.py:450-584)."""

    class ObjectiveStatusReporter:
        REPORTABLES = {"pop_best", "pop_best_eval", "mean_eval", "median_eval"}

        def __init__(self, algorithm: SearchAlgorithm, *, obj_index: int, to_report: str):
            if to_report not in self.REPORTABLES:
                raise ValueError(f"Unrecognized report request: {to_report}")
            self._algorithm, self._obj_index, self._to_report = algorithm, int(obj_index), to_report

        @property
        def population(self) -> SolutionBatch:
            return self._algorithm.population

        def _get_pop_best(self):
            return self.population[int(self.population.argbest(self._obj_index))].clone()

        def _get_pop_best_eval(self):
            for key in ("pop_best", f"obj{self._obj_index}_pop_best"):
                if self._algorithm.has_status_key(key):
                    best = self._algorithm.get_status_value(key)
                    if best is not None and best.is_evaluated:
                        return float(best.evals[self._obj_index])
            return None

        @torch.no_grad()
        def _get_mean_eval(self):
            return float(torch.mean(self.population.access_evals(self._obj_index)))

        @torch.no_grad()
        def _get_median_eval(self):
            return float(torch.median(self.population.access_evals(self._obj_index)))

        def __call__(self):
            return getattr(self, "_get_" + self._to_report)()

    def __init__(self, *, exclude: Optional[Iterable] = None, enable: bool = True):
        if not enable:
            return
        reporter = self.ObjectiveStatusReporter
        excluded = set() if exclude is None else set(exclude)
        single_obj: Optional[int] = None
        if getattr(self, "obj_index", None) is not None:
            single_obj = self.obj_index
        elif len(self.problem.senses) == 1:
            single_obj = 0
        if single_obj is not None:
            for name in reporter.REPORTABLES - excluded:
                self.add_status_getters({name: reporter(self, obj_index=single_obj, to_report=name)})
        else:
            for i_obj in range(len(self.problem.senses)):
                for name in reporter.REPORTABLES - excluded:
                    self.add_status_getters({f"obj{i_obj}_{name}": reporter(self, obj_index=i_obj, to_report=name)})
