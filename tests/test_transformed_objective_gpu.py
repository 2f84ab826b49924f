"""Objectives of the transformed row y = M (x - o) on the GPU: both paths against the float64 torch function, the exact zero at
y = 0, permutations bit for bit against the untransformed kernels, the ask's noise, isolation of items, 70 000 items without
host synchronisation, the routing of every ask-and-evaluate path, and a search-level check that the transform reaches the search."""

import importlib.util
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, ops
    from evotorch_b200.algorithms import CMAES
    from evotorch_b200.algorithms.functional import (cem, cem_ask_and_evaluate, cmaes, cmaes_ask_and_evaluate, cmaes_tell, pgpe,
                                                     pgpe_ask_and_evaluate, sepcmaes, sepcmaes_ask_and_evaluate, sepcmaes_tell)
    from evotorch_b200.algorithms.functional.misc import draw_philox_seed
    from evotorch_b200.objectives import FusedObjective

DEV = "cuda"
CUTOFF = 96  # EVOK_TRANSFORM_FUSED_MAX_D: the largest D of the fused path
DIMS = [1, 2, 3, 4, 5, 31, 32, 33, CUTOFF - 1, CUTOFF, CUTOFF + 1, 500, 1000, 2048]


def _load(filename):
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), filename)
    spec = importlib.util.spec_from_file_location("_" + filename[:-3], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


T = _load("test_transformed_objective.py")


def _transform(batch, D, seed, kind="rotation"):
    M, o = T.transform(batch, D, torch.Generator().manual_seed(seed), kind)
    return M.to(DEV), o.to(DEV)


# ------------------------------------------------------------------------------------------------ values
@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("per_item", [False, True])
def test_values_against_float64(D, per_item):
    """Every objective of the CPU tests, on the path of its D, against its torch function in float64 on the float32 rows.  With an
    orthogonal M each y_j is a sum of D products of size |x - o| <= 10, so float32 (the FMA chain or 3xTF32) errs by about
    sqrt(D) 2^-24 |x - o| per entry; every f here is a sum of positive terms or 10 D plus bounded terms, far from 0, so a relative
    1e-4 covers it with margin at D = 2048.  The general M of Rastrigin has condition 10 and |y| <= 100: 5e-4 relative."""
    B, n = (5, 7) if D <= 500 else (3, 5)
    gen = torch.Generator().manual_seed(D)
    for name in T.SPECS:
        kind = "general" if name == "rot_rastrigin" else "rotation"
        M, o = _transform((B,) if per_item else (), D, D * 7 + per_item, kind)
        obj, _ = T.make(name, M, o, gen)
        X = (o.unsqueeze(-2) + (torch.rand(B, n, D, generator=gen) * 6 - 3).to(DEV)).contiguous()
        got = obj.evaluate_batched(X)
        ref = obj(X.double())
        rtol = 5e-4 if kind == "general" else 1e-4
        torch.testing.assert_close(got.double(), ref, rtol=rtol, atol=1e-3 if name == "rot_schwefel_1_2" and D == 1 else 1e-6,
                                   msg=lambda m: f"{name} D={D} per_item={per_item}: {m}")
        assert torch.equal(obj(X), got)  # obj(values) runs the same kernels


@pytest.mark.parametrize("D", [3, 10, CUTOFF, CUTOFF + 1, 1000])
def test_row_at_offset_gives_value_at_zero(D):
    """A row equal to o has y = 0 exactly on both paths, whatever M: the ellipsoid of condition 1e6 is then exactly 0, even with a
    scaled M and |o| up to 4 (a GEMM of X M^T - M o would not be)."""
    B = 3
    M, o = _transform((B,), D, D, "general")
    obj, _ = T.make("rot_ellipsoid", M * 100, o, torch.Generator().manual_seed(0))
    X = o[:, None, :].expand(B, 5, D).contiguous()
    assert torch.equal(obj.evaluate_batched(X), torch.zeros(B, 5, device=DEV))


@pytest.mark.parametrize("D", [3, 32, 33, 64, CUTOFF])
@pytest.mark.parametrize("name", ["rot_ellipsoid", "rot_rosenbrock", "rot_schwefel_1_2", "rot_rastrigin"])
def test_permutation_is_bit_exact_on_fused_path(D, name):
    """With M a permutation (or the identity) and o = 0, the fused path folds the permuted row in eval_row's order: the bits of the
    untransformed objective's batched evaluation of the permuted rows."""
    B, n = 3, 9
    gen = torch.Generator().manual_seed(D)
    X = torch.randn(B, n, D, generator=gen).to(DEV) * 3
    twin = FusedObjective(name + "_twin", **T.twin_keywords(name))
    for perm in (torch.arange(D), torch.randperm(D, generator=gen)):
        P = torch.eye(D)[perm].to(DEV)  # y_j = x_perm[j]
        obj = FusedObjective(name, transform=P, **T.SPECS[name][0])
        assert torch.equal(obj.evaluate_batched(X), twin.evaluate_batched(X[..., perm.to(DEV)].contiguous()))


# ------------------------------------------------------------------------------------------------ noise
def test_ask_noise_and_element_noise():
    D, B = 12, 5
    M, o = _transform((B,), D, 3)
    obj = FusedObjective("noisy", sums={"s": "(y + 0.1 * randn())**2 + 0.01 * rand()"}, value="s + rand()", transform=(M, o))
    state = cmaes(center_init=torch.zeros(B, D, device=DEV), stdev_init=1.0, objective_sense="min")
    torch.manual_seed(11)
    values, evals = cmaes_ask_and_evaluate(state, objective=obj)
    torch.manual_seed(11)
    seed = draw_philox_seed()  # the ask's z draw
    assert torch.equal(evals, obj.evaluate_batched(values, seed=seed))
    sstate = sepcmaes(center_init=torch.zeros(B, D, device=DEV), stdev_init=1.0, objective_sense="min")
    torch.manual_seed(12)
    values, evals = sepcmaes_ask_and_evaluate(sstate, objective=obj)
    torch.manual_seed(12)
    assert torch.equal(evals, obj.evaluate_batched(values, seed=draw_philox_seed()))
    # the element and value noise of the untransformed kernel for the same key: the identity transform on the fused path
    eye = FusedObjective("noisy_eye", sums={"s": "(y + 0.1 * randn())**2 + 0.01 * rand()"}, value="s + rand()", transform=torch.eye(D, device=DEV))
    twin = FusedObjective("noisy_twin", sums={"s": "(x + 0.1 * randn())**2 + 0.01 * rand()"}, value="s + rand()")
    X = torch.randn(B, 9, D, device=DEV)
    assert torch.equal(eye.evaluate_batched(X, seed=77), twin.evaluate_batched(X, seed=77))


def test_noise_free_evaluation_draws_no_key():
    """Like an untransformed objective, a transformed one without noise takes no Philox key: obj(X) and evaluate_batched leave
    torch's generator where it was, so a run on it draws the host numbers its untransformed twin draws."""
    M, o = _transform((), 12, 17)
    obj, _ = T.make("rot_ellipsoid", M, o, torch.Generator().manual_seed(0))
    X = torch.randn(4, 6, 12, device=DEV)
    state = torch.get_rng_state()
    obj(X[0]), obj(X), obj.evaluate_batched(X)
    assert torch.equal(torch.get_rng_state(), state)


# ------------------------------------------------------------------------------------------------ isolation, scale, sync
@pytest.mark.parametrize("D", [7, 300])
def test_nonfinite_item_changes_no_other(D):
    B, n = 5, 6
    M, o = _transform((B,), D, 5)
    obj, _ = T.make("rot_rastrigin", M, o, torch.Generator().manual_seed(1))
    X = torch.randn(B, n, D, device=DEV)
    clean = obj.evaluate_batched(X)
    for what in ("X", "M", "o"):
        Xp, Mp, op = (t.clone(memory_format=torch.contiguous_format) for t in (X, M, o))
        {"X": Xp, "M": Mp, "o": op}[what][2].view(-1)[::3] = float("nan")
        {"X": Xp, "M": Mp, "o": op}[what][3].view(-1)[0] = float("inf")
        got = obj.with_data(transform=(Mp, op)).evaluate_batched(Xp)
        keep = [0, 1, 4]
        assert torch.equal(got[keep], clean[keep]), what


@pytest.mark.parametrize("D", [8, 200])
def test_many_items_no_sync_and_fixed_launches(D):
    B = 70_000 if D == 8 else 1000
    n = 5
    M, o = _transform((), D, 9)
    obj, _ = T.make("rot_ellipsoid", M, o, torch.Generator().manual_seed(2))
    X = torch.randn(B, n, D, device=DEV)
    f = obj.evaluate_batched(X, seed=1)
    idx = torch.tensor([0, 1, B // 2, B - 1], device=DEV)
    torch.testing.assert_close(f[idx].double(), obj(X[idx].double()), rtol=1e-4, atol=1e-6)
    counts = []
    for b in (3, 17, 101):
        Xb = X[:b].contiguous()
        obj.evaluate_batched(Xb, seed=1)  # warm: workspace and module
        torch.cuda.synchronize()
        before = ops.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            obj.evaluate_batched(Xb, seed=1)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append(ops.launch_count() - before)
    assert counts[0] == counts[1] == counts[2] >= 1


def test_gemm_path_chunk_seams():
    """Past 256 MB of x - o and y the GEMM path runs item chunks: at D = 200 and n = 400 an item takes 2 * 400 * 200 * 4 bytes, so
    a chunk is 419 items and 900 items are three chunks.  Items on both sides of each seam, each with its own M, o, data and noise
    stream, get the bits of a call on that item alone with stream id b (noise), and the float64 torch function (data)."""
    D, n, B = 200, 400, 900
    chunk = (256 << 20) // (2 * n * D * 4)
    assert chunk == 419
    M, o = _transform((B,), D, 21)
    M = M.contiguous()
    X = (o[:, None, :] + torch.randn(B, n, D, device=DEV)).contiguous()
    seams = [0, chunk - 1, chunk, 2 * chunk - 1, 2 * chunk, B - 1]
    noisy = FusedObjective("noisy_seams", sums={"s": "(y + 0.01 * randn())**2"}, value="s + rand()", transform=(M, o))
    f = noisy.evaluate_batched(X, seed=5)
    for b in seams:
        one = ops.evaluate_transform_batched(noisy._transform_id, X[b:b + 1], M[b:b + 1], o[b:b + 1], seed=5, stream_id0=b)
        assert torch.equal(one[0], f[b]), b
    lun, _ = T.make("lunacek_like", M, o, torch.Generator().manual_seed(4))
    got = lun.evaluate_batched(X)
    ref = lun(X.double())
    idx = torch.tensor(seams, device=DEV)
    torch.testing.assert_close(got[idx].double(), ref[idx], rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------------ routing
def test_every_ask_and_evaluate_path_evaluates_transformed_values():
    D, B = 6, 4
    M, o = _transform((B,), D, 13)
    obj, _ = T.make("rot_ellipsoid", M, o, torch.Generator().manual_seed(3))
    center = torch.zeros(B, D, device=DEV)
    for values, evals in (pgpe_ask_and_evaluate(pgpe(center_init=center, center_learning_rate=0.1, stdev_learning_rate=0.1,
                                                     objective_sense="min", stdev_init=1.0), popsize=10, objective=obj),
                          cem_ask_and_evaluate(cem(center_init=center, parenthood_ratio=0.5, objective_sense="min", stdev_init=1.0),
                                               popsize=10, objective=obj),
                          cmaes_ask_and_evaluate(cmaes(center_init=center, stdev_init=1.0, objective_sense="min"), objective=obj),
                          sepcmaes_ask_and_evaluate(sepcmaes(center_init=center, stdev_init=1.0, objective_sense="min"), objective=obj)):
        assert isinstance(values, torch.Tensor)
        torch.testing.assert_close(evals.double(), obj(values.double()), rtol=1e-4, atol=1e-6)
    with pytest.raises(ValueError, match="transformed row"):
        pgpe_ask_and_evaluate(pgpe(center_init=center, center_learning_rate=0.1, stdev_learning_rate=0.1, objective_sense="min",
                                  stdev_init=1.0), popsize=10, objective=obj, lazy=True)
    with pytest.raises(ValueError, match="transformed row"):
        sepcmaes_ask_and_evaluate(sepcmaes(center_init=center, stdev_init=1.0, objective_sense="min"), objective=obj, lazy=True)
    shared, _ = T.make("rot_ellipsoid", M[0], o[0], torch.Generator().manual_seed(3))
    with pytest.raises(ValueError, match="transformed row"):
        Problem("min", shared, solution_length=D, initial_bounds=(-1, 1), device=DEV, lazy_population=True)
    prob = Problem("min", shared, solution_length=D, initial_bounds=(-1, 1), device=DEV, seed=0)
    searcher = CMAES(prob, stdev_init=1.0, popsize=12)
    searcher.step()
    pop = searcher.population
    torch.testing.assert_close(pop.evals[:, 0].double(), shared(pop.values.double()), rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------------ search level
def _share(obj, family, B, D, gens, tau):
    state = (cmaes if family == "full" else sepcmaes)(center_init=torch.zeros(B, D, device=DEV), stdev_init=3.0, objective_sense="min")
    ask, tell = (cmaes_ask_and_evaluate, cmaes_tell) if family == "full" else (sepcmaes_ask_and_evaluate, sepcmaes_tell)
    best = torch.full((B,), math.inf, device=DEV)
    for _ in range(gens):
        values, evals = ask(state, objective=obj)
        state = tell(state, values, evals)
        best = torch.fmin(best, evals.min(-1).values)  # fmin: a converged search's later NaN rows do not erase its best
    return (best < tau).float().mean().item()


def test_rotation_reaches_the_search():
    """Rotated ellipsoid of condition 1e6, D = 10, 256 items, |o| up to 4.  The thresholds come from a float64 run of the torch path
    with 64 items (scripts/transformed_search_calibration.py, output in results/transformed_search_calibration.json): every
    full-covariance search was below 1e-4 by generation 500, rotated and unrotated, every separable one by 200 on the unrotated
    twin, and no separable one on the rotated ellipsoid in 1200.  So: G = 600, tau = 1e-4 (400 float32 ulps of f at the optimum,
    about 2.5e-7 each), and a share of at least 0.9 where the family fits, at most 0.1 where it does not."""
    B, D, G, tau = 256, 10, 600, 1e-4
    torch.manual_seed(0)
    R = torch.linalg.qr(torch.randn(B, D, D, dtype=torch.float64))[0].float().to(DEV)
    o = (8 * torch.rand(B, D) - 4).to(DEV)
    rotated = FusedObjective("rot_ell", sums={"s": T.ELLIPSOID}, value="s", transform=(R, o))
    twin = rotated.with_data(transform=(torch.eye(D, device=DEV).expand(B, D, D).contiguous(), o))
    shares = {(f, k): _share(obj, f, B, D, G, tau) for f in ("full", "sep") for k, obj in (("rot", rotated), ("unrot", twin))}
    print("success shares", shares)
    assert shares["full", "rot"] >= 0.9 and shares["full", "unrot"] >= 0.9 and shares["sep", "unrot"] >= 0.9
    assert shares["sep", "rot"] <= 0.1
