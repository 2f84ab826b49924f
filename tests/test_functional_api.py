"""Functional ask/tell API (SURVEY 8 f2) against golden vectors produced by the real reference
(tests/golden/gen_functional_golden.py -> functional_golden.npz).  CPU tests exercise the generic path and the host logic;
the `gpu` tests replay the same tells through the kernels."""

import os

import numpy as np
import pytest
import torch

from evotorch_b200.algorithms import functional as F

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "functional_golden.npz"))
DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


def T(x, device):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32, device=device)


OPT_CASES = {
    "clipup": (F.clipup, F.clipup_ask, F.clipup_tell, dict(center_learning_rate=0.15, momentum=0.9),
               lambda dev: dict(center_learning_rate=T([0.1, 0.2, 0.3], dev), max_speed=T([0.15, 0.5, 0.45], dev))),
    "adam": (F.adam, F.adam_ask, F.adam_tell, dict(center_learning_rate=0.05),
             lambda dev: dict(center_learning_rate=T([0.01, 0.05, 0.1], dev), beta1=0.8)),
    "sgd": (F.sgd, F.sgd_ask, F.sgd_tell, dict(center_learning_rate=0.1, momentum=0.5),
            lambda dev: dict(center_learning_rate=T([0.1, 0.2, 0.3], dev))),
}


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("name", list(OPT_CASES))
@pytest.mark.parametrize("tag", ["plain", "batched"])
def test_functional_optimizers_match_reference(name, tag, device):
    init, ask, tell, cfg, cfg_b = OPT_CASES[name]
    start = GOLD["opt/c0"] if tag == "plain" else GOLD["opt/c0_b"]
    grads = GOLD["opt/grads"] if tag == "plain" else GOLD["opt/grads_b"]
    state = init(center_init=T(start, device), **(cfg if tag == "plain" else cfg_b(device)))
    first = state
    for g, want in zip(grads, GOLD[f"opt/{name}/{tag}/centers"]):
        state = tell(state, follow_grad=T(g, device))
        np.testing.assert_allclose(ask(state).cpu().numpy(), want, rtol=2e-6, atol=2e-6)
    # functional: the old state is untouched
    np.testing.assert_array_equal(ask(first).cpu().numpy(), start)


PGPE_CASES = {
    "sym_clipup": dict(center_learning_rate=0.3, stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0),
    "nonsym_adam_nes": dict(center_learning_rate=0.05, stdev_learning_rate=0.1, objective_sense="min", stdev_init=0.7, optimizer="adam",
                            ranking_method="nes", symmetric=False, stdev_max_change=None),
    "sym_sgd_linear_max": dict(center_learning_rate=0.1, stdev_learning_rate=0.2, objective_sense="max", radius_init=3.0, optimizer="sgd",
                               ranking_method="linear", stdev_min=0.5, stdev_max=1.0, stdev_max_change=0.1),
    "batched": dict(center_learning_rate=[0.2, 0.4], stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0),
}


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("tag", list(PGPE_CASES))
def test_functional_pgpe_tell_matches_reference(tag, device):
    kw = dict(PGPE_CASES[tag])
    if tag == "batched":
        kw["center_learning_rate"] = T(kw["center_learning_rate"], device)
    state = F.pgpe(center_init=T(GOLD[f"pgpe/{tag}/center0"], device), **kw)
    np.testing.assert_allclose(state.stdev.cpu().numpy(), GOLD[f"pgpe/{tag}/stdev0"], rtol=1e-6)
    for g in range(GOLD[f"pgpe/{tag}/values"].shape[0]):
        state = F.pgpe_tell(state, T(GOLD[f"pgpe/{tag}/values"][g], device), T(GOLD[f"pgpe/{tag}/evals"][g], device))
        np.testing.assert_allclose(state.optimizer_state.center.cpu().numpy(), GOLD[f"pgpe/{tag}/center"][g], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(state.stdev.cpu().numpy(), GOLD[f"pgpe/{tag}/stdev"][g], rtol=1e-5, atol=1e-5)


CEM_CASES = {
    "plain": dict(parenthood_ratio=0.25, objective_sense="min", stdev_init=2.0, stdev_max_change=0.3),
    "max_bounds": dict(parenthood_ratio=0.5, objective_sense="max", stdev_init=1.0, stdev_min=0.4, stdev_max=1.5),
    "batched": dict(parenthood_ratio=0.25, objective_sense="min"),
    # the edges, where the reference gives NaN: one elite (std of one row), no elite, a zero stdev with an unlimited max change
    "one_elite": dict(parenthood_ratio=0.03, objective_sense="min", stdev_init=1.0),
    "zero_elites": dict(parenthood_ratio=0.01, objective_sense="max", stdev_init=1.0),
    "zero_stdev": dict(parenthood_ratio=0.25, objective_sense="min"),
}


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("tag", list(CEM_CASES))
def test_functional_cem_tell_matches_reference(tag, device):
    kw = dict(CEM_CASES[tag])
    if tag in ("batched", "zero_stdev"):
        kw["stdev_init"] = T(GOLD[f"cem/{tag}/stdev0"], device)
    state = F.cem(center_init=T(GOLD[f"cem/{tag}/center0"], device), **kw)
    for g in range(GOLD[f"cem/{tag}/values"].shape[0]):
        state = F.cem_tell(state, T(GOLD[f"cem/{tag}/values"][g], device), T(GOLD[f"cem/{tag}/evals"][g], device))
        np.testing.assert_allclose(state.center.cpu().numpy(), GOLD[f"cem/{tag}/center"][g], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(state.stdev.cpu().numpy(), GOLD[f"cem/{tag}/stdev"][g], rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize("device", DEVICES)
def test_functional_ask_shapes_statistics_and_seeding(device):
    torch.manual_seed(5)
    center = T(np.linspace(-2, 2, 24).reshape(2, 12), device)
    state = F.pgpe(center_init=center, center_learning_rate=0.1, stdev_learning_rate=0.1, objective_sense="min",
                   stdev_init=T([[0.5] * 12, [2.0] * 12], device))
    pop = F.pgpe_ask(state, popsize=4000)
    assert pop.shape == (2, 4000, 12) and pop.device.type == device
    # antithetic pairs mirror around the centre; the two batch items are different draws with their own centre / stdev
    torch.testing.assert_close(pop[:, 0::2] + pop[:, 1::2], (2 * center)[:, None, :].expand(2, 2000, 12), rtol=0, atol=1e-5)
    eps = (pop[:, 0::2] - center[:, None, :])
    np.testing.assert_allclose(eps.std(dim=1).cpu().numpy(), np.stack([np.full(12, 0.5), np.full(12, 2.0)]), rtol=0.08)
    assert not torch.allclose(eps[0] / 0.5, eps[1] / 2.0)
    torch.manual_seed(5)
    assert torch.equal(F.pgpe_ask(state, popsize=4000), pop)  # torch.manual_seed reproduces the ask
    assert not torch.equal(F.pgpe_ask(state, popsize=4000), pop)
    with pytest.raises(ValueError):
        F.pgpe_ask(state, popsize=33)
    cst = F.cem(center_init=center[0], parenthood_ratio=0.5, objective_sense="min", stdev_init=1.0)
    assert F.cem_ask(cst, popsize=33).shape == (33, 12)


@pytest.mark.parametrize("device", DEVICES)
def test_functional_pgpe_optimises_and_validates(device):
    torch.manual_seed(1)
    state = F.pgpe(center_init=torch.full((20,), 3.0, device=device), center_learning_rate=0.3, stdev_learning_rate=0.1,
                   objective_sense="min", stdev_init=1.0)
    first = None
    for _ in range(40):
        pop = F.pgpe_ask(state, popsize=200)
        f = (pop**2).sum(-1)
        first = float(f.mean()) if first is None else first
        state = F.pgpe_tell(state, pop, f)
    assert float(f.mean()) < 0.2 * first
    with pytest.raises(ValueError):
        F.pgpe(center_init=torch.zeros(4), center_learning_rate=0.1, stdev_learning_rate=0.1, objective_sense="minimise", stdev_init=1.0)
    with pytest.raises(ValueError):
        F.pgpe(center_init=torch.zeros(4), center_learning_rate=0.1, stdev_learning_rate=0.1, objective_sense="min")
    with pytest.raises(ValueError):
        F.pgpe(center_init=torch.zeros(4), center_learning_rate=0.1, stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0, radius_init=2.0)
    with pytest.raises(ValueError):
        F.pgpe(center_init=torch.zeros(4), center_learning_rate=0.1, stdev_learning_rate=0.1, objective_sense="min", stdev_init=[1.0, 2.0])
    with pytest.raises(ValueError):
        F.get_functional_optimizer("rmsprop")
    with pytest.raises(ValueError):
        F.clipup(center_init=torch.zeros(3))
    triple = F.get_functional_optimizer((F.sgd, F.sgd_ask, F.sgd_tell))
    assert triple.initialize is F.sgd and triple.tell is F.sgd_tell
