"""Leaving and re-entering CUDA-graph mode: a searcher that is re-captured while a graph exists (`enable_cuda_graph()` again),
then steps eagerly (`enable_cuda_graph(False)`) and then captures once more (`True`) must follow a never-graphed run bit for bit,
and the problem's device-side generation counter (`philox_stream_offset`) is attached only while a graph is being captured."""

import pytest
import torch

from evotorch_b200 import Problem
from evotorch_b200.algorithms import CMAES, PGPE, SNES
from evotorch_b200.objectives import rastrigin

pytestmark = pytest.mark.gpu

DEV = "cuda"
GENERATIONS = 12
# generation -> `enable_cuda_graph` argument given right before it: re-capture with a graph in place, leave graph mode, come back
SWITCHES = {4: True, 7: False, 9: True}
CASES = ["pgpe", "pgpe_lazy", "snes", "cmaes_full", "sepcma", "sepcma_lazy"]


def _make(case):
    prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=160, device=DEV, seed=13,
                   lazy_population=case.endswith("_lazy"))
    if case.startswith("pgpe"):
        return PGPE(prob, popsize=600, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    if case == "snes":
        return SNES(prob, popsize=600, stdev_init=2.0)
    if case == "cmaes_full":
        return CMAES(prob, stdev_init=1.0, popsize=256, limit_C_decomposition=False)
    return CMAES(prob, stdev_init=1.0, popsize=600, separable=True)


def _state(s):
    if isinstance(s, CMAES):
        return {"m": s.m, "sigma": s.sigma, "C": s.C, "A": s.A, "evals": s.population.evals, "values": s.population.values}
    return {"center": s.status["center"], "stdev": s.status["stdev"], "evals": s.population.evals, "values": s.population.values}


@pytest.mark.parametrize("case", CASES)
def test_leaving_and_reentering_graph_mode_matches_eager(case):
    eager, graph = _make(case), _make(case).enable_cuda_graph()
    for g in range(GENERATIONS):
        if g in SWITCHES:
            graph.enable_cuda_graph(SWITCHES[g])
        eager.step()
        graph.step()
        assert graph.problem.philox_stream_offset is None, g
        a, b = _state(eager), _state(graph)
        for key in a:
            assert torch.equal(a[key], b[key]), (g, key)
        assert graph.problem._philox_stream == eager.problem._philox_stream, g
        if g in (3, 6, GENERATIONS - 1):
            assert graph._graph is not None, g
        if g in (7, 8):
            assert graph._graph is None, g
