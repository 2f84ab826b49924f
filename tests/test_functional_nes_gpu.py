"""Functional XNES and SNES on the kernels: the exponential pair against scipy in float64, the XNES tell against the float64 oracle
and the reference golden, bits (item b against a one-item call, the ask against `cmaes_ask`'s draw, repeated runs), 70 000 items and
launches per generation, no host synchronisation, NaN isolation, fused objectives through the ask, SNES stored against lazy and
against the object-API arithmetic, and the search outcome on a rotated ellipsoid."""

import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import ops
    from evotorch_b200.algorithms.functional import (cmaes, cmaes_ask, snes, snes_ask, snes_ask_and_evaluate, snes_tell, xnes, xnes_ask,
                                                     xnes_ask_and_evaluate, xnes_tell)
    from evotorch_b200.algorithms.functional.misc import draw_philox_seed
    from evotorch_b200.distributions import ExpSeparableGaussian
    from evotorch_b200.objectives import FusedObjective, rastrigin
    from evotorch_b200.tools import modify_tensor
from oracle import functional_nes_oracle as O

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_golden.npz"))


def random_symmetric(B, D, norm2, seed):
    """(B, D, D) float32 symmetric matrices Q diag(lam) Q^T with max |lam| = norm2 (the 2-norm)."""
    g = torch.Generator().manual_seed(seed)
    Q = torch.linalg.qr(torch.randn(B, D, D, generator=g, dtype=torch.float64))[0]
    lam = 2 * torch.rand(B, D, generator=g, dtype=torch.float64) - 1
    lam = lam / lam.abs().amax(-1, keepdim=True) * norm2
    S = (Q * lam[:, None, :]) @ Q.mT
    return (0.5 * (S + S.mT)).float()


def expm_errors(D, norm2, B=4, seed=0):
    """(largest Frobenius error of F+ and F- relative to |F64|, F+, F-, S): the kernel against scipy's expm(+-S) - I of the float32 S."""
    import scipy.linalg

    S = random_symmetric(B, D, norm2, seed)
    Fp, Fm = ops.sym_expm_pair_batched(S.to(DEV))
    Fp, Fm = Fp.double().cpu().numpy(), Fm.double().cpu().numpy()
    eye = np.eye(D)
    errs = []
    for b in range(B):
        s = S[b].double().numpy()
        Ep, Em = scipy.linalg.expm(s), scipy.linalg.expm(-s)
        for F, E in ((Fp[b], Ep), (Fm[b], Em)):
            ref = E - eye
            errs.append(np.linalg.norm(F - ref) / max(np.linalg.norm(ref), 1e-300))
    return max(errs), Fp, Fm, S


@pytest.mark.parametrize("D", [1, 2, 17, 64, 96])
@pytest.mark.parametrize("norm2", [0.0, 1e-7, 1e-3, 0.5, 4.0, 40.0])
def test_expm_pair_against_scipy(D, norm2):
    """Frobenius error <= 1e-5 |F64| for |S|_2 <= 1 (the expm1 form keeps a tiny S's relative precision) and <= 1e-4 |F64| above,
    F64 = expm(+-S) - I in float64; and (I + F-)(I + F+) = I, the inverse pair, where the product is representable.  Above
    |S|_2 = 1 the error is not measured against |expm(+-S)|: where every eigenvalue of +-S is far below 0, expm(+-S) lies below
    the float32 resolution of I, which F = expm(+-S) - I carries."""
    err, Fp, Fm, S = expm_errors(D, norm2)
    if norm2 == 0.0:
        assert np.all(Fp == 0) and np.all(Fm == 0)
        return
    assert err <= (1e-5 if norm2 <= 1 else 1e-4), err
    if norm2 <= 4:
        eye = np.eye(D)
        for b in range(len(S)):
            P = (eye + Fm[b]) @ (eye + Fp[b])
            assert np.linalg.norm(P - eye) <= 1e-5 * np.linalg.norm(eye + Fm[b]) * np.linalg.norm(eye + Fp[b])


def _state(B, D, seed, popsize=None, method="nes", lr=0.3, cond=3.0):
    """A float32 CUDA XNES state with random centres and well-conditioned random A (singular values in [1/cond, cond])."""
    g = torch.Generator().manual_seed(seed)
    Q = torch.linalg.qr(torch.randn(B, D, D, generator=g, dtype=torch.float64))[0]
    A = (Q * torch.exp(math.log(cond) * (2 * torch.rand(B, 1, D, generator=g, dtype=torch.float64) - 1))).float()
    s = xnes(center_init=torch.randn(B, D, generator=g).to(DEV), stdev_init=1.0, objective_sense="min", popsize=popsize, ranking_method=method,
             stdev_learning_rate=lr, scale_learning_rate=False)
    return s._replace(A=A.to(DEV).contiguous(), A_inv=torch.linalg.inv(A.double()).float().to(DEV).contiguous())


def _numpy(*ts):
    return tuple(t.double().cpu().numpy() for t in ts)


@pytest.mark.parametrize("D", [5, 33, 96])
@pytest.mark.parametrize("method", ["nes", "centered"])
def test_tell_against_oracle(D, method):
    s = _state(6, D, seed=D, method=method)
    torch.manual_seed(D)
    x = xnes_ask(s)
    f = (x * x * torch.linspace(1, 10, D, device=DEV)).sum(-1)
    s1 = xnes_tell(s, x, f)
    mu, A, A_inv = O.xnes_tell(*_numpy(s.center, s.A, s.A_inv, x, f), maximize=False, ranking=method, lr_mu=1.0, lr_A=0.3)
    for got, ref in ((s1.center, mu), (s1.A, A), (s1.A_inv, A_inv)):
        got = got.double().cpu().numpy()
        assert np.abs(got - ref).max() <= 2e-5 * np.abs(ref).max() * max(1.0, math.sqrt(D) / 4), np.abs(got - ref).max()


@pytest.mark.parametrize("method", ["nes", "centered"])
def test_tell_against_reference_golden(golden, method):
    mu, A, A_inv = (torch.tensor(golden[f"xnes/{k}"], device=DEV)[None] for k in ("mu", "A", "A_inv"))
    X, f = torch.tensor(golden["xnes/X"], device=DEV)[None], torch.tensor(golden["xnes/f"], device=DEV)[None]
    s = xnes(center_init=mu, stdev_init=1.0, objective_sense="min", popsize=X.shape[1], ranking_method=method, stdev_learning_rate=0.3,
             scale_learning_rate=False)._replace(A=A, A_inv=A_inv)
    s1 = xnes_tell(s, X, f)
    close = lambda a, k, atol: np.testing.assert_allclose(a[0].cpu().numpy(), golden[f"xnes/{method}/{k}"], rtol=2e-5, atol=atol)  # noqa: E731
    close(s1.center, "new_mu", 3e-6)
    close(s1.A, "new_A", 3e-6)
    close(s1.A_inv, "new_A_inv", 6e-6)


def test_item_bits_and_expm_item_bits():
    B, D = 9, 21
    s = _state(B, D, seed=1)
    torch.manual_seed(3)
    x = xnes_ask(s)
    f = (x * x).sum(-1)
    w = ops.rank_batched(f, "nes", False)
    ops.weights_adjust_batched_(w, 1)
    outs = ops.xnes_tell_batched(x, w, s.center, s.A, s.A_inv, 1.0, 0.3)
    S = random_symmetric(B, D, 3.0, 2).to(DEV)
    Fp, Fm = ops.sym_expm_pair_batched(S)
    for b in range(B):
        sl = slice(b, b + 1)
        one = ops.xnes_tell_batched(x[sl], w[sl], s.center[sl], s.A[sl], s.A_inv[sl], 1.0, 0.3)
        assert all(torch.equal(o[b], p[0]) for o, p in zip(outs, one))
        p1, m1 = ops.sym_expm_pair_batched(S[sl])
        assert torch.equal(Fp[b], p1[0]) and torch.equal(Fm[b], m1[0])


def test_ask_is_cmaes_draw_path():
    """Under the same seed, xnes_ask draws the z of cmaes_ask and maps them through the same GEMM: same bits."""
    B, D = 5, 12
    s = _state(B, D, seed=2)
    c = cmaes(center_init=s.center, stdev_init=1.0, objective_sense="min", popsize=s.popsize)._replace(A=s.A)
    torch.manual_seed(5)
    a = xnes_ask(s)
    torch.manual_seed(5)
    assert torch.equal(a, cmaes_ask(c))


def _gen(s, obj=None):
    v, e = xnes_ask_and_evaluate(s, objective=obj or rastrigin)
    return xnes_tell(s, v, e)


def test_repeated_run_bits():
    runs = []
    for _ in range(2):
        s = xnes(center_init=torch.full((7, 10), 2.0, device=DEV), stdev_init=1.0, objective_sense="min")
        torch.manual_seed(11)
        for _ in range(20):
            s = _gen(s)
        runs.append(s)
    for name in ("center", "A", "A_inv"):
        assert torch.equal(getattr(runs[0], name), getattr(runs[1], name)), name


def test_70000_items_and_launches_per_generation():
    B, D = 70000, 4
    s = _state(B, D, seed=4)
    torch.manual_seed(1)
    x = xnes_ask(s)
    f = (x * x).sum(-1)
    w = ops.rank_batched(f, "nes", False)
    ops.weights_adjust_batched_(w, 1)
    outs = ops.xnes_tell_batched(x, w, s.center, s.A, s.A_inv, 1.0, 0.3)
    S = random_symmetric(B, D, 2.0, 3).to(DEV)
    Fp, _ = ops.sym_expm_pair_batched(S)
    for b in (0, 65534, 65535, 69999):
        sl = slice(b, b + 1)
        one = ops.xnes_tell_batched(x[sl], w[sl], s.center[sl], s.A[sl], s.A_inv[sl], 1.0, 0.3)
        assert all(torch.equal(o[b], p[0]) for o, p in zip(outs, one))
        assert torch.equal(ops.sym_expm_pair_batched(S[sl])[0][0], Fp[b])
    counts = []
    for B in (1, 37, 4000):
        st = xnes(center_init=torch.zeros(B, 16, device=DEV), stdev_init=1.0, objective_sense="min")
        st = _gen(st)
        before = ops.launch_count()
        _gen(st)
        torch.cuda.synchronize()
        counts.append(ops.launch_count() - before)
    assert counts[0] == counts[1] == counts[2], counts


def test_no_host_synchronisation():
    obj = FusedObjective("nes_sync_sphere", sums={"s": "x**2"}, value="s")
    s = xnes(center_init=torch.ones(8, 20, device=DEV), stdev_init=1.0, objective_sense="min")
    n = snes(center_init=torch.ones(8, 200, device=DEV), stdev_init=1.0, objective_sense="min", stdev_max_change=0.2)
    for _ in range(2):
        s = _gen(s, obj)
        v, e = snes_ask_and_evaluate(n, objective=obj, lazy=True)
        n = snes_tell(n, v, e)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            s = _gen(s, obj)
            v, e = snes_ask_and_evaluate(n, objective=obj, lazy=True)
            n = snes_tell(n, v, e)
            v, e = snes_ask_and_evaluate(n, objective=obj)
            n = snes_tell(n, v, e)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_nan_isolation():
    """NaN and inf in other items' rows and state leave item 0's bits alone, and give non-finite results only where they are."""
    B, D = 4, 30
    s = _state(B, D, seed=6)
    torch.manual_seed(2)
    x = xnes_ask(s)
    f = (x * x).sum(-1)
    w = ops.rank_batched(f, "nes", False)
    ops.weights_adjust_batched_(w, 1)
    ref = ops.xnes_tell_batched(x, w, s.center, s.A, s.A_inv, 1.0, 0.3)
    x2, A2, mu2 = x.clone(), s.A.clone(), s.center.clone()
    x2[1, 3] = float("nan")
    A2[2, 0, 0] = float("inf")
    mu2[3] = float("nan")
    out = ops.xnes_tell_batched(x2, w, mu2, A2, s.A_inv, 1.0, 0.3)
    for o, r in zip(out, ref):
        assert torch.equal(o[0], r[0])
    assert not torch.isfinite(out[1][1]).all() and not torch.isfinite(out[1][3]).all()
    S = random_symmetric(3, D, 1.0, 4).to(DEV)
    Fp, Fm = ops.sym_expm_pair_batched(S)
    S[1, 2, 2] = float("nan")
    S[2, 0, 1] = float("inf")
    Fp2, Fm2 = ops.sym_expm_pair_batched(S)
    assert torch.equal(Fp2[0], Fp[0]) and torch.equal(Fm2[0], Fm[0])
    assert not torch.isfinite(Fp2[1]).all() and not torch.isfinite(Fp2[2]).all()


def test_objectives_through_the_ask():
    """Built-in, transformed, per-item-data and noisy FusedObjectives get the ask's Philox seed through xnes_ask_and_evaluate."""
    B, D = 3, 24
    s = _state(B, D, seed=9)
    g = torch.Generator().manual_seed(0)
    R = torch.linalg.qr(torch.randn(B, D, D, generator=g, dtype=torch.float64))[0].float().to(DEV)
    o = torch.randn(B, D, generator=g).to(DEV)
    objs = [FusedObjective("nes_rot", sums={"s": "10**(2 * j / (D - 1)) * y**2"}, value="s", transform=(R, o)),
            FusedObjective("nes_rot_noisy", sums={"s": "y**2"}, value="s + 0.1 * randn()", transform=(R, o)),
            FusedObjective("nes_shifted", sums={"s": "(x - o)**2"}, value="s", data={"o": o}),
            FusedObjective("nes_noisy", sums={"s": "x**2 + 0.01 * randn()"}, value="s")]
    for obj in objs:
        torch.manual_seed(21)
        v, e = xnes_ask_and_evaluate(s, objective=obj)
        torch.manual_seed(21)
        seed = draw_philox_seed()
        assert torch.equal(e, obj.evaluate_batched(v, seed=seed))
        assert torch.isfinite(e).all() and e.shape == (B, s.popsize)
    v, e = xnes_ask_and_evaluate(s, objective=rastrigin)
    torch.testing.assert_close(e, rastrigin(v), rtol=1e-5, atol=1e-4)
    v2, e2 = xnes_ask_and_evaluate(s, objective=objs[2])
    torch.testing.assert_close(e2, ((v2 - o[:, None, :]) ** 2).sum(-1), rtol=1e-5, atol=1e-4)


def test_snes_lazy_equals_stored_bits():
    runs = {}
    for lazy in (False, True):
        n = snes(center_init=torch.full((5, 300), 3.0, device=DEV), stdev_init=1.0, objective_sense="min", stdev_max_change=0.2, stdev_min=0.01)
        torch.manual_seed(4)
        for _ in range(6):
            v, e = snes_ask_and_evaluate(n, objective=rastrigin, lazy=lazy)
            n = snes_tell(n, v, e)
        runs[lazy] = n
    assert torch.equal(runs[False].center, runs[True].center) and torch.equal(runs[False].stdev, runs[True].stdev)


@pytest.mark.parametrize("method", ["nes", "centered"])
def test_snes_against_object_arithmetic(method):
    """B items against B ExpSeparableGaussian updates (the arithmetic of B `SNES` objects) on the same populations."""
    B, D = 6, 50
    n = snes(center_init=torch.randn(B, D, device=DEV), stdev_init=torch.rand(B, D, device=DEV) + 0.5, objective_sense="min",
             ranking_method=method, stdev_max_change=0.1, center_learning_rate=0.9)
    torch.manual_seed(8)
    x = snes_ask(n)
    f = rastrigin(x)
    n1 = snes_tell(n, x, f)
    for b in range(B):
        dist = ExpSeparableGaussian({"mu": n.center[b], "sigma": n.stdev[b]})
        grads = dist.compute_gradients(x[b], f[b], objective_sense="min", ranking_method=method)
        upd = dist.update_parameters(grads, learning_rates={"mu": 0.9, "sigma": n.stdev_learning_rate})
        sig = modify_tensor(n.stdev[b], upd.sigma, max_change=n.stdev_max_change)
        torch.testing.assert_close(n1.center[b], upd.mu, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(n1.stdev[b], sig, rtol=1e-5, atol=1e-6)


# results/functional_nes_calibration.json (float64 torch path, 32 items, rotated ellipsoid of condition 1e4 at D = 16): the share
# of XNES items with f < 1e-6 by each generation, and no SNES item by 5000.  The test asks for 90 % of the XNES items within the
# budget below: every item succeeds by generation 2000 in the calibration (none by 1500), and 500 more allow for float32.
SEARCH_BUDGET = 2500


def test_search_outcome():
    import importlib.util

    path = os.path.join(ROOT, "scripts", "functional_nes_calibration.py")
    spec = importlib.util.spec_from_file_location("_nes_calibration", path)
    C = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(C)
    B = 32
    obj = C.problem(B, device=DEV)
    torch.manual_seed(0)
    xn = C.shares("xnes", obj, B, (SEARCH_BUDGET,), dtype=torch.float32, device=DEV)[SEARCH_BUDGET]
    sn = C.shares("snes", obj, B, (SEARCH_BUDGET,), dtype=torch.float32, device=DEV)[SEARCH_BUDGET]
    assert xn >= 0.9 and sn <= 0.1, (xn, sn)
