"""evotorch_b200: the per-generation hot path of EvoTorch's distribution-based searchers (PGPE / SNES / CEM / XNES /
CMA-ES) as hand-written sm_90a (H100) CUDA kernels behind the reference's Problem / SolutionBatch / SearchAlgorithm API.

    from evotorch_b200 import Problem
    from evotorch_b200.algorithms import PGPE
    from evotorch_b200.objectives import rastrigin

    problem = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=10_000, device="cuda", seed=0)
    searcher = PGPE(problem, popsize=100_000, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    searcher.run(100)
"""

from . import algorithms, distributions, logging, neuroevolution, objectives, optimizers, testing, tools
from .core import Problem, Solution, SolutionBatch

__version__ = "0.1.0"
__all__ = ["Problem", "Solution", "SolutionBatch", "algorithms", "distributions", "logging", "neuroevolution", "objectives", "optimizers", "testing", "tools"]
