"""NEProblem / SupervisedNE against golden fitnesses produced by the REAL reference's one-solution-at-a-time loop
(tests/golden/gen_ne_golden.py; neproblem.py:407-429, supervisedne.py:327-347), through the batched route of this package;
CPU here, CUDA (kernel path: K8 / tensor-core GEMM) when a GPU is present."""

import os

import numpy as np
import pytest
import torch
from torch import nn
from torch.utils.data import TensorDataset

from evotorch_b200 import SolutionBatch
from evotorch_b200.algorithms import PGPE, SNES
from evotorch_b200.neuroevolution import NEProblem, SupervisedNE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVICES = ["cpu", "cuda"]


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(ROOT, "tests", "golden", "ne_golden.npz")) as z:
        return {k: z[k] for k in z.files}


def _net(dims, act):
    return nn.Sequential(nn.Linear(int(dims[0]), int(dims[1])), act(), nn.Linear(int(dims[1]), int(dims[2])))


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("tag,act", [("mlp_tanh", nn.Tanh), ("mlp_relu_wide", nn.ReLU)])
def test_supervisedne_matches_reference_losses(gold, tag, act, device):
    X, Y, P = (torch.as_tensor(gold[f"supervised/{tag}/{k}"]) for k in ("X", "Y", "P"))
    dims = gold[f"supervised/{tag}/dims"]
    for loss, key, kw in ((nn.MSELoss(), "loss", dict(num_minibatches=2)), (lambda yh, y: torch.mean(torch.abs(yh - y)), "l1", {})):
        prob = SupervisedNE(TensorDataset(X, Y), lambda: _net(dims, act), loss, minibatch_size=len(X), common_minibatch=True, device=device, **kw)
        assert prob.solution_length == P.shape[1]
        batch = SolutionBatch(prob, len(P))
        batch.set_values(P.to(device))
        prob.evaluate(batch)
        assert prob._batched_ok  # the whole population went through batched_forward, not the per-solution loop
        np.testing.assert_allclose(batch.evals[:, 0].cpu().numpy(), gold[f"supervised/{tag}/{key}"], rtol=2e-5, atol=1e-6)
        # the reference's own loop (one network at a time) on the same problem object gives the same numbers
        prob._batched_ok = False
        batch2 = SolutionBatch(prob, len(P))
        batch2.set_values(P.to(device))
        prob.evaluate(batch2)
        np.testing.assert_allclose(batch2.evals[:, 0].cpu().numpy(), gold[f"supervised/{tag}/{key}"], rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize("device", DEVICES)
def test_neproblem_matches_reference_evaluations(gold, device):
    probe = torch.as_tensor(gold["neproblem/probe"]).to(device)

    def evaluator(net):
        y = net(probe)
        return torch.sum(y * y), torch.stack([y.mean(), y.max()])

    prob = NEProblem("max", nn.Sequential(nn.Linear(5, 7), nn.Tanh(), nn.Linear(7, 2)), evaluator, eval_data_length=2, device=device)
    assert prob.solution_length == int(gold["neproblem/solution_length"][0]) and prob.network_device == torch.device(device)
    P = torch.as_tensor(gold["neproblem/P"]).to(device)
    batch = SolutionBatch(prob, len(P))
    batch.set_values(P)
    prob.evaluate(batch)
    np.testing.assert_allclose(batch.evals.cpu().numpy(), gold["neproblem/evals"], rtol=2e-5, atol=1e-6)
    net = prob.make_net(P[3])
    np.testing.assert_allclose(net(probe).detach().cpu().numpy(), gold["neproblem/make_net_out"], rtol=2e-5, atol=1e-6)
    assert net is not prob.parameterize_net(P[0])  # make_net copies, parameterize_net fills THE network
    # batched_forward == row-by-row parameterize_net
    yb = prob.batched_forward(P, probe)
    for i in (0, 5, 11):
        np.testing.assert_allclose(yb[i].cpu().numpy(), prob.parameterize_net(P[i])(probe).detach().cpu().numpy(), rtol=2e-5, atol=1e-6)


def test_reference_examples_run_unchanged():
    """tests/test_examples.py:80-231 of the reference: the NEProblem and SupervisedNE quick-starts."""
    from evotorch_b200.tools import device_of, dtype_of

    def sign_prediction_score(network: torch.nn.Module):
        samples = torch.randn((32, 3), dtype=dtype_of(network), device=device_of(network))
        sign_out = torch.sign(network(samples)[:, 0])
        sign_sum = torch.sign(samples.sum(dim=-1))
        return ((sign_sum == sign_out).to(torch.float).sum() - (sign_sum != sign_out).to(torch.float).sum()) / 32

    problem = NEProblem(objective_sense="max", network=torch.nn.Linear(3, 1), network_eval_func=sign_prediction_score)
    searcher = PGPE(problem, popsize=10, radius_init=2.25, center_learning_rate=0.2, stdev_learning_rate=0.1)
    searcher.run(2)
    assert "best" in searcher.status and searcher.step_count == 2

    N = 100
    X = torch.randn((N, 2))
    Y = X.sum(dim=-1, keepdim=True)
    for network in (nn.Sequential(nn.Linear(2, 32), nn.ReLU(), nn.Linear(32, 1)), lambda: nn.Sequential(nn.Linear(2, 32), nn.ReLU(), nn.Linear(32, 1)),
                    "Linear(2, 32) >> ReLU() >> Linear(32, 1)"):
        sum_of_problem = SupervisedNE(dataset=TensorDataset(X, Y), network=network, minibatch_size=32, loss_func=nn.MSELoss())
        searcher = SNES(sum_of_problem, popsize=50, radius_init=2.25)
        searcher.run(2)
        assert "best" in searcher.status and searcher.step_count == 2
    # non-common minibatches and subclassing keep the per-solution loop of the reference
    class Custom(SupervisedNE):
        def _loss(self, y_hat, y):
            return torch.mean((y_hat - y) ** 2)

    c = Custom(TensorDataset(X, Y), nn.Linear(2, 1), minibatch_size=16, common_minibatch=False)
    s = SNES(c, popsize=12, radius_init=1.0)
    s.run(2)
    assert s.step_count == 2
