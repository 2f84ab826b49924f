"""The Philox draw of a population (`PhiloxDraw`): what `Problem.next_philox_draw()` captures, the rule that keys the population
between two generations under a CUDA graph, and the gradient input of a lazy population.  CPU only: the kernels that consume a
draw are covered by test_gpu_kernels.py, test_grad_hybrid.py, test_sepcma.py and test_generation_graph.py."""

import pytest
import torch

from evotorch_b200 import Problem
from evotorch_b200.core import LazySolutionBatch, PhiloxDraw
from evotorch_b200.objectives import rastrigin


def _problem() -> Problem:
    return Problem("min", rastrigin, initial_bounds=(-1, 1), solution_length=8, lazy_population=True, seed=3)


def test_next_philox_draw_advances_the_stream_by_one_and_captures_row0_and_offset():
    prob = _problem()
    prob._philox_stream = 41
    first = prob.next_philox_draw()
    assert (first.seed, first.stream_id, first.row0, first.stream_offset) == (prob._philox_seed, 41, 0, None)
    assert prob._philox_stream == 42

    counter = torch.zeros(1, dtype=torch.int32)
    prob.philox_row0, prob.philox_stream_offset = 6, counter
    second = prob.next_philox_draw()
    prob.philox_row0, prob.philox_stream_offset = 0, None  # changed after the draw: the draw keeps what it captured
    assert (second.seed, second.stream_id, second.row0) == (prob._philox_seed, 42, 6)
    assert second.stream_offset is counter
    assert prob._philox_stream == 43
    assert second.kwargs == dict(seed=prob._philox_seed, stream_id=42, row0=6, stream_offset=counter)
    with pytest.raises(AttributeError):
        second.stream_id = 0  # a draw is a value


def test_between_generations_is_the_identity_eagerly_and_one_stream_lower_under_a_graph():
    eager = PhiloxDraw(7, 5, 4)
    assert eager.between_generations() is eager

    counter = torch.zeros(1, dtype=torch.int32)
    graphed = PhiloxDraw(7, 5, 4, counter)
    prev = graphed.between_generations()
    assert (prev.seed, prev.stream_id, prev.row0) == (7, 4, 4)
    assert prev.stream_offset is counter
    assert graphed.stream_id == 5


def test_lazy_batch_answers_gradient_samples_with_its_recipe_without_materialising():
    prob = _problem()
    batch = LazySolutionBatch(prob, 4)
    mu, sigma = torch.zeros(8), torch.ones(8)
    recipe = PhiloxDraw(1, 2).recipe(4, True, mu, sigma)
    assert recipe.shape == (4, 8)

    def materialize(*args, **kwargs):
        raise AssertionError("the gradient input of a lazy population must not regenerate the N x D values")

    recipe.materialize = materialize
    batch.recipe = recipe
    assert batch.gradient_samples(mu, sigma) is recipe
