"""BASELINE config 1 shape (the reference README's SNES: popsize 1000, dim 100, Rastrigin) on one GPU: generations/s with
eager stepping and with CUDA-graph replay."""
import json
import sys
import time

import torch

sys.path.insert(0, ".")
from evotorch_b200 import Problem  # noqa: E402
from evotorch_b200.algorithms import PGPE, SNES  # noqa: E402
from evotorch_b200.objectives import rastrigin  # noqa: E402


def run(make, graph, steps=2000):
    s = make()
    if graph:
        s.enable_cuda_graph()
    for _ in range(20):
        s.step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        s.step()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


for name, make in (("SNES 1000 x 100", lambda: SNES(Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=100, device="cuda", seed=1), popsize=1000, stdev_init=10.0)),
                   ("PGPE 1000 x 100", lambda: PGPE(Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=100, device="cuda", seed=1), popsize=1000,
                                                    center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)),
                   ("PGPE 10000 x 1000", lambda: PGPE(Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=1000, device="cuda", seed=1), popsize=10000,
                                                      center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0))):
    print(json.dumps({"config": name, "eager_generations_per_s": round(run(make, False), 1), "graph_generations_per_s": round(run(make, True), 1)}), flush=True)
