"""Functional (explicit-state, ask/tell) counterparts of the distribution-based searchers and their optimizers
(reference: evotorch/algorithms/functional/__init__.py).  Every function accepts extra leftmost batch dimensions.

    state = pgpe(center_init=x0, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0, objective_sense="min")
    for _ in range(generations):
        population = pgpe_ask(state, popsize=1000)
        state = pgpe_tell(state, population, f(population))
    best_guess = state.optimizer_state.center

Full-covariance CMA-ES over a batch of independent searches (one launch per stage for all of them on CUDA float32):

    state = cmaes(center_init=torch.randn(1024, 32, device="cuda"), stdev_init=1.0, objective_sense="min")
    for _ in range(generations):
        population = cmaes_ask(state)                        # (1024, popsize, 32)
        state = cmaes_tell(state, population, f(population))

With an objective that has a fused kernel, `pgpe_ask_and_evaluate` / `cem_ask_and_evaluate` sample and evaluate all batch items
in one launch, and with `lazy=True` never store the population:

    population, evals = pgpe_ask_and_evaluate(state, popsize=1000, objective=rastrigin, lazy=True)
    state = pgpe_tell(state, population, evals)

`cmaes_ask_and_evaluate` evaluates the full-covariance asks of all items in one launch of the batched evaluation kernel, keyed
with the ask's Philox draw, so per-item data and noise reach CMA-ES too:

    population, evals = cmaes_ask_and_evaluate(state, objective=shifted_sphere)   # data of batch shape (1024,)
    state = cmaes_tell(state, population, evals)

`restarts` wraps a `cmaes` or `sepcmaes` state for multi-start search: per item, best-ever tracking, termination criteria and
re-initialisation on the device, each item with its own generation counter:

    rs = restarts(state, lb=-5.0, ub=5.0)
    values, evals = cmaes_ask_and_evaluate(rs.search, objective=rastrigin)
    rs = restarts_tell(rs, values, evals)                # rs.best_values, rs.best_evals, rs.num_restarts, rs.stop_flags

With `restarts(state, ..., popsize_multiplier=2, max_popsize=640)` every restart of an item doubles its population size (IPOP):
the ask draws 640 rows per item and item b uses its first `rs.popsize[b]`.  With `bipop=True` as well, restarts alternate between
that ladder and small runs of random population size and step size, each regime given a similar share of the evaluations (BIPOP).

LM-MA-ES learns rotations at solution lengths where `cmaes` cannot hold its D x D matrices: each item keeps m ~ 4 + 3 ln D
direction vectors, O(m D) state and work per sample, and a fixed number of launches per generation for all items:

    state = lmmaes(center_init=torch.zeros(8, 100_000, device="cuda"), stdev_init=1.0, objective_sense="min")
    for _ in range(generations):
        population, evals = lmmaes_ask_and_evaluate(state, objective=rotated)   # (8, popsize, 100_000), (8, popsize)
        state = lmmaes_tell(state, population, evals)

XNES and SNES, the natural evolution strategies, run many searches at once too.  On CUDA float32 the XNES tell is one CTA per
item for D <= 96 (its exponential map included), and SNES takes `lazy=True` like `pgpe`:

    state = xnes(center_init=torch.randn(1024, 16, device="cuda"), stdev_init=1.0, objective_sense="min")
    for _ in range(generations):
        population, evals = xnes_ask_and_evaluate(state, objective=rastrigin)   # (1024, popsize, 16), (1024, popsize)
        state = xnes_tell(state, population, evals)

    state = snes(center_init=torch.zeros(64, 10_000, device="cuda"), stdev_init=1.0, objective_sense="min")
    population, evals = snes_ask_and_evaluate(state, objective=rastrigin, lazy=True)
    state = snes_tell(state, population, evals)
"""

from .funcadam import AdamState, adam, adam_ask, adam_tell
from .funccem import CEMState, cem, cem_ask, cem_ask_and_evaluate, cem_tell
from .funcclipup import ClipUpState, clipup, clipup_ask, clipup_tell
from .funccmaes import CMAESState, cmaes, cmaes_ask, cmaes_ask_and_evaluate, cmaes_tell
from .funclmmaes import LMMAESState, lmmaes, lmmaes_ask, lmmaes_ask_and_evaluate, lmmaes_tell
from .funcpgpe import PGPEState, pgpe, pgpe_ask, pgpe_ask_and_evaluate, pgpe_tell
from .funcrestarts import IPOPLadder, RestartState, bipop_ladder, ipop_ladder, restarts, restarts_tell
from .fused import LazyPopulation
from .funcsepcmaes import SepCMAESState, sepcmaes, sepcmaes_ask, sepcmaes_ask_and_evaluate, sepcmaes_tell
from .funcsgd import SGDState, sgd, sgd_ask, sgd_tell
from .funcsnes import SNESState, snes, snes_ask, snes_ask_and_evaluate, snes_tell
from .funcxnes import XNESState, xnes, xnes_ask, xnes_ask_and_evaluate, xnes_tell
from .misc import OptimizerFunctions, get_functional_optimizer

__all__ = ["AdamState", "adam", "adam_ask", "adam_tell", "CEMState", "cem", "cem_ask", "cem_ask_and_evaluate", "cem_tell", "ClipUpState",
           "clipup", "clipup_ask", "clipup_tell", "CMAESState", "cmaes", "cmaes_ask", "cmaes_ask_and_evaluate", "cmaes_tell", "LazyPopulation",
           "LMMAESState", "lmmaes", "lmmaes_ask", "lmmaes_ask_and_evaluate", "lmmaes_tell", "PGPEState", "pgpe", "pgpe_ask", "pgpe_ask_and_evaluate", "pgpe_tell",
           "IPOPLadder", "RestartState", "bipop_ladder", "ipop_ladder", "restarts", "restarts_tell",
           "SepCMAESState", "sepcmaes", "sepcmaes_ask", "sepcmaes_ask_and_evaluate", "sepcmaes_tell",
           "SGDState", "sgd", "sgd_ask", "sgd_tell", "SNESState", "snes", "snes_ask", "snes_ask_and_evaluate", "snes_tell",
           "XNESState", "xnes", "xnes_ask", "xnes_ask_and_evaluate", "xnes_tell", "OptimizerFunctions", "get_functional_optimizer"]
