"""Whole-generation CUDA graphs: the one capture-and-replay protocol shared by every searcher that replays a generation."""

from __future__ import annotations

from typing import Callable

import torch

from .. import _native as nat
from .. import ops
from ..core import Problem


class GenerationGraph:
    """One generation of a searcher captured into a CUDA graph; `replay()` runs the next generation.

    The body takes its draw as an eager step does (`problem.next_philox_draw()`) and hands it to every kernel that samples or
    regenerates the population.  While the capture runs, `problem.philox_stream_offset`, and so the draw's `stream_offset`, is a
    fresh device-side int32 generation counter, zero until the first replay and incremented by the graph after the body, so the
    k-th replay (k = 0, 1, ...) draws from stream `base + k`, `base` being the host stream id the capture started from;
    `replay()` advances the host counter alongside.  The population that exists between two generations is therefore keyed
    `(base - 1) + counter` (`PhiloxDraw.between_generations()`): read while replay k runs, the counter is k and that is the
    previous replay's population, the one the body consumes; read after it, the counter is k + 1 and that is the population
    replay k drew.  Outside the capture the attribute is None again: the graph reads the counter through the pointer it baked
    in, and an eager step after any number of replays continues on the next host stream id.  Every capture allocates its own
    counter, because a lazy population's `PhiloxRecipe` may still reference the one of an earlier graph.

    The body runs under `private_workspaces()`, so the graph owns the scratch buffers it writes to.  `buffers` are tensors made
    outside the capture that nothing but the graph uses any more: the graph keeps them alive, because its kernels read and write
    them through baked-in pointers.  The body itself is not kept (it usually refers to the searcher that holds this graph)."""

    def __init__(self, problem: Problem, body: Callable[[], None], *, buffers: tuple = ()):
        self.problem, self.buffers = problem, buffers
        self.counter = torch.zeros(1, dtype=torch.int32, device=problem.device)
        self.graph = torch.cuda.CUDAGraph()
        base = problem._philox_stream
        problem.philox_stream_offset = self.counter
        before = ops.launch_count()
        try:
            with nat.private_workspaces() as self.workspaces, torch.cuda.graph(self.graph):
                body()
                self.counter.add_(1)
        finally:
            problem.philox_stream_offset = None
            problem._philox_stream = base  # the capture consumed host-side stream ids without running anything
        self.kernels = ops.launch_count() - before  # kernels of libevok.so inside one replay
        ops.count_replayed_launches(-self.kernels)  # the capture itself executed none of them

    def replay(self):
        self.graph.replay()
        ops.count_replayed_launches(self.kernels)
        self.problem._philox_stream += 1
