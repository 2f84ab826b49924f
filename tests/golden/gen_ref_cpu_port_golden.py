"""Golden vectors of tests/test_ref_cpu_port.py::test_port_is_bit_identical_to_the_reference: the real reference's PGPE run
(Rastrigin, dim 300, popsize 200, seed 5, 8 generations).  Run with the reference importable as `evotorch`:

    PYTHONPATH=tests/golden/_refstubs:<reference checkout>/src EVOTORCH_VERBOSE_LEVEL=0 python tests/golden/gen_ref_cpu_port_golden.py

Stores center and stdev after every generation and the population of the first and the last generation (float32, exact).
"""

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import evotorch  # noqa: E402
from evotorch import Problem  # noqa: E402
from evotorch.algorithms import PGPE  # noqa: E402

from oracle.ref_cpu_path import rastrigin  # noqa: E402

assert not evotorch.__file__.startswith(os.path.dirname(os.path.dirname(HERE))), "import the reference, not this package"
prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=300, vectorized=True, seed=5, dtype=torch.float32)
s = PGPE(prob, popsize=200, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
mu, sigma, X = [], [], {}
for t in range(8):
    s.step()
    mu.append(s.status["center"].numpy().copy())
    sigma.append(s.status["stdev"].numpy().copy())
    if t in (0, 7):
        X[t] = s.population.values.numpy().copy()
np.savez_compressed(os.path.join(HERE, "ref_cpu_port_golden.npz"), mu=np.stack(mu), sigma=np.stack(sigma), X_first=X[0], X_last=X[7])
print("wrote", os.path.join(HERE, "ref_cpu_port_golden.npz"))
