"""FusedObjective with noise on the GPU: the draws of every sampling path against the numpy restatement (oracle/noise_oracle.py),
bit-identity between the paths that must agree, independence of the draws, and the refusal of an evaluation without a key."""

import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from oracle import es_oracle as O
from oracle import noise_oracle as N

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import _native as nat
    from evotorch_b200 import ops

DEV = "cuda"
SEED, SID = 0x5EED_0000_1234_5678, 11
Z_TOL = 5e-5  # the sampler's z against the float64 Box-Muller (tests/test_gpu_kernels.py)


def _load(filename):
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), filename)
    spec = importlib.util.spec_from_file_location("_" + filename[:-3], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CPU = _load("test_noisy_objective.py")
_objs = {}


def obj(name):
    if name not in _objs:
        _objs[name] = CPU.make(name)
    return _objs[name]


def same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def params(D, offset=False):
    g = torch.Generator().manual_seed(D)
    mu = (torch.rand(D + offset, generator=g) - 0.5).to(DEV)[offset:]
    sg = (0.5 + torch.rand(D + offset, generator=g)).to(DEV)[offset:]
    return mu, sg


def sample(name, n, D, symmetric, lazy=False, offset=False, row0=0, stream_id=SID):
    mu, sg = params(D, offset)
    X = None if lazy else torch.empty(n, D, device=DEV)
    f = torch.empty(n, device=DEV)
    ops.sample_eval(obj(name).evok_objective_id, X, mu, sg, n_rows=n, symmetric=symmetric, seed=SEED, stream_id=stream_id, row0=row0, f=f)
    return X, f, mu, sg


def rows(n, row0=0):
    return np.arange(row0, row0 + n, dtype=np.uint64)


@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
def test_value_draws_against_the_oracle(symmetric, lazy, offset):
    n, D = 256, 36
    _, f, _, _ = sample("value_rand", n, D, symmetric, lazy, offset, row0=64)
    assert np.array_equal(f.cpu().numpy().astype(np.float64), N.value_noise(SEED, SID, rows(n, 64), 4, False))  # bit for bit
    _, f, _, _ = sample("value_randn", n, D, symmetric, lazy, offset)
    assert np.abs(f.cpu().numpy() - N.value_noise(SEED, SID, rows(n), 4, True)).max() < Z_TOL


def _element_reference(name, X, row0=0):
    Xd = X.double().cpu().numpy()
    n, D = Xd.shape
    if name == "elem_rand":
        u = N.element_noise(SEED, SID, rows(n, row0), D, 0, False)
        return u.sum(1), np.abs(u).sum(1) * 2.0**-23 * D
    z = N.element_noise(SEED, SID, rows(n, row0), D, 0, True)
    t = (Xd + z) ** 2
    return t.sum(1), (t.sum(1) * 2.0**-22 * (D + 4) + 2 * np.abs(Xd + z).sum(1) * Z_TOL)


@pytest.mark.parametrize("name", ["elem_rand", "elem_randn"])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("D", [1, 3, 4, 5, 127, 128, 129, 260, 1000, 1028, 10_001])
def test_element_draws_within_the_float64_bound(D, symmetric, name):
    for offset in (False, True):
        X, f, _, _ = sample(name, 64, D, symmetric, offset=offset)
        ref, bound = _element_reference(name, X)
        err = np.abs(f.double().cpu().numpy() - ref)
        assert (err <= bound + 1e-6).all(), (D, offset, float((err / (bound + 1e-6)).max()))


def test_f7_and_bbob_against_the_oracle():
    n, D = 128, 260
    X, f, _, _ = sample("f7", n, D, True)
    Xd = X.double().cpu().numpy()
    ref = ((np.arange(D) + 1) * Xd**4).sum(1) + N.value_noise(SEED, SID, rows(n), 4, False)
    assert np.allclose(f.cpu().numpy(), ref, rtol=1e-5, atol=1e-5)
    X, f, _, _ = sample("bbob_rastrigin", n, D, False)
    Xd = X.double().cpu().numpy()
    ref = (10 * D + (Xd**2 - 10 * np.cos(2 * np.pi * Xd)).sum(1)) * np.exp(0.01 * N.value_noise(SEED, SID, rows(n), 4, True))
    assert np.allclose(f.cpu().numpy(), ref, rtol=1e-4, atol=1e-3)


# ------------------------------------------------------------------------------------------------ keyed evaluation
# 1 .. 5: one partial group; 127 .. 132 and 255 .. 260: step boundaries and ragged tails; 388 / 516: the 4-group step of the
# vectorised path; 512 / 1028: the 128-group warp steps; 10 001: several of each with a scalar tail
EVAL_DIMS = [1, 3, 4, 5, 127, 128, 129, 132, 255, 260, 388, 512, 516, 1000, 1028, 4096, 10_000, 10_001]
EVAL_NAMES = ["value_rand", "elem_rand_j", "elem_randn", "running_pair_noise"]
E = 2.0**-24


def keyed_reference(name, Xd, row0=0, mutate=False):
    """(float64 fitness, first-order bound) of the rows Xd (global rows row0 ..) under the draw (SEED, SID); mutate: the same
    noise with the two columns of every word pair swapped (a wrong word / z0-z1 choice), which must fall outside the bound."""
    n, D = Xd.shape
    K = math.ceil(D / 32) + 12  # adds along a lane (at most ceil(D / 32) terms each), 5 butterfly rounds, spare
    r = rows(n, row0)

    def elem(k, normal):
        u = N.element_noise(SEED, SID, r, D, k, normal)
        if mutate:
            u = u[:, np.arange(D) ^ 1 if D % 2 == 0 else np.r_[np.arange(D - 1) ^ 1, D - 1]]
        return u

    if name == "value_rand":
        return N.value_noise(SEED, SID, r, 4, False), np.zeros(n)
    if name == "elem_rand_j":
        t = (np.arange(D) + 1) * elem(0, False)
        return t.sum(1), E * (K + 1) * np.abs(t).sum(1)
    if name == "elem_randn":
        z = elem(0, True)
        t = (Xd + z) ** 2
        return t.sum(1), E * (K + 3) * t.sum(1) + 2 * (np.abs(Xd + z) * Z_TOL).sum(1)
    # running_pair_noise: s = sum_j c_j z_j with c_j = sum_{k<=j} x_k, p = sum_j (x_{j+1} - x_j)^2, value s + p + randn()
    z = elem(0, True)
    c = np.cumsum(Xd, 1)
    err_c = E * (12 + np.arange(D) / 32) * np.cumsum(np.abs(Xd), 1)
    ts = c * z
    tp = np.diff(Xd, axis=1) ** 2
    v = N.value_noise(SEED, SID, r, 4, True)
    S, P = ts.sum(1), tp.sum(1)
    bound = ((np.abs(z) * err_c + np.abs(c) * Z_TOL).sum(1) + E * (K + 2) * np.abs(ts).sum(1) + E * (K + 4) * tp.sum(1) + Z_TOL
             + 3 * E * (np.abs(S) + P + np.abs(v)))
    return S + P + v, bound


@pytest.mark.parametrize("name", EVAL_NAMES)
@pytest.mark.parametrize("D", EVAL_DIMS)
def test_keyed_evaluation_against_the_oracle_and_the_sampler(D, name):
    """evaluate_keyed on the vectorised path (aligned X, D % 4 == 0) and the scalar path (X at a column offset), against the
    float64 oracle on the same x, and bit for bit against the sampler where both take the vectorised path."""
    n, row0 = 96, 1000
    o = obj(name)
    X, fs, _, _ = sample(name, n, D, False, row0=row0)
    Xd = X.double().cpu().numpy()
    ref, bound = keyed_reference(name, Xd, row0)
    wide = torch.zeros(n, D + 1, device=DEV)
    wide[:, 1:] = X  # column offset 1: a row stride and a base that are not 16-byte aligned, the scalar path
    for label, Xe in (("aligned", X), ("offset", wide[:, 1:])):
        fe = ops.evaluate_keyed(o.evok_objective_id, Xe, seed=SEED, stream_id=SID, row0=row0)
        got = fe.double().cpu().numpy()
        if name == "value_rand":
            assert np.array_equal(got, ref), label  # bit for bit
        else:
            err = np.abs(got - ref)
            assert (err <= bound).all(), (label, float((err / np.maximum(bound, 1e-30)).max()))
            if 128 <= D <= 1028:  # the bound tells a wrong word of the draw apart (it grows faster than the effect with D)
                mref, _ = keyed_reference(name, Xd, row0, mutate=True)
                assert (np.abs(got - mref) > bound).any(), label
    if D % 4 == 0:
        fe = ops.evaluate_keyed(o.evok_objective_id, X, seed=SEED, stream_id=SID, row0=row0)
        assert same(fe, fs)


@pytest.mark.parametrize("name", ["input_noise_sphere", "where_noise", "running_pair_noise", "f7"])
@pytest.mark.parametrize("symmetric", [True, False])
def test_bit_identities_between_paths(name, symmetric):
    n, D = 512, 260
    X, f, mu, sg = sample(name, n, D, symmetric)
    _, fl, _, _ = sample(name, n, D, symmetric, lazy=True)
    assert same(f, fl)  # lazy == stored
    half = n // 2  # a launch split at row0 (sharding) == one launch
    f2 = torch.empty(n, device=DEV)
    oid = obj(name).evok_objective_id
    for r0 in (0, half):
        ops.sample_eval(oid, None, mu, sg, n_rows=half, symmetric=symmetric, seed=SEED, stream_id=SID, row0=r0, f=f2[r0:r0 + half])
    assert same(f, f2)
    fe = ops.evaluate_keyed(oid, X, seed=SEED, stream_id=SID)  # the keyed evaluation on the VEC path == the sampler
    assert same(f, fe)
    fe2 = ops.evaluate_keyed(oid, X[half:], seed=SEED, stream_id=SID, row0=half)
    assert same(f[half:], fe2)
    if not symmetric:  # the squared-norm sampler of separable CMA-ES
        q, fq = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        ops.sample_eval_sq(oid, None, mu, sg, q, n_rows=n, f=fq, seed=SEED, stream_id=SID)
        assert same(f, fq)


@pytest.mark.parametrize("symmetric", [True, False])
def test_batched_items_are_single_launches_on_their_streams(symmetric):
    o = obj("input_noise_sphere")
    o.compile_batched()
    B, n, D = 5, 64, 132
    g = torch.Generator().manual_seed(3)
    mu = torch.randn(B, D, generator=g).to(DEV)
    sg = (0.5 + torch.rand(B, D, generator=g)).to(DEV)
    f = torch.empty(B, n, device=DEV)
    ops.sample_eval_batched(o.evok_objective_id, None, mu, sg, f, symmetric=symmetric, seed=SEED, stream_id0=SID)
    for b in range(B):
        fb = torch.empty(n, device=DEV)
        ops.sample_eval(o.evok_objective_id, None, mu[b].contiguous(), sg[b].contiguous(), n_rows=n, symmetric=symmetric, seed=SEED,
                        stream_id=SID + b, f=fb)
        assert same(f[b], fb), b


def test_push_variant_at_two_simulated_ranks():
    pw = _load("test_peer_exchange_world.py")
    counts, D = [64, 64], 132
    world = pw.SimWorld(counts, D)
    mu, sg = params(D)
    o = obj("where_noise")
    world.poison()
    for r, px in enumerate(world.px):
        with world.on(r):
            ops.sample_eval_push(o.evok_objective_id, None, mu, sg, n_rows=counts[r], symmetric=True, seed=SEED, stream_id=SID,
                                 row0=world.row0[r], peer=px)
    world.producers_done()
    for r, px in enumerate(world.px):
        with world.on(r):
            px.wait_fitness()
    _, f, _, _ = sample("where_noise", sum(counts), D, True)
    torch.cuda.synchronize()
    for px in world.px:
        assert same(px.f_all, f)


def test_element_occurrences_and_the_population_z_are_uncorrelated():
    """Two element occurrences at the same (row, column), and each against the z of that element: column 2 of D = 4 picked out
    by where(j == 2, ...), read through two objectives that differ only in which occurrence `value` returns."""
    sums = {"a": "where(j == 2, randn(), 0)", "b": "where(j == 2, rand(), 0)"}
    from evotorch_b200.objectives import FusedObjective

    oa, ob = FusedObjective("occurrence_a", sums=sums, value="a"), FusedObjective("occurrence_b", sums=sums, value="b")
    n, D = 1 << 20, 4
    zero, one = torch.zeros(D, device=DEV), torch.ones(D, device=DEV)
    X = torch.empty(n, D, device=DEV)
    fa, fb = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    for o, f in ((oa, fa), (ob, fb)):
        ops.sample_eval(o.evok_objective_id, X, zero, one, n_rows=n, symmetric=False, seed=SEED, stream_id=SID, f=f)
    z = X[:, 2].double()  # x = 0 + 1 * z
    # the sampler's Box-Muller (fast lg2 / sqrt / sincos): within Z_TOL on the bulk, and less accurate far in the tails, which
    # 2^20 rows reach
    err = np.abs(fa.double().cpu().numpy() - N.element_noise(SEED, SID, rows(n), D, 0, True)[:, 2])
    assert np.quantile(err, 0.999) < Z_TOL and err.max() < 1e-3
    assert np.array_equal(fb.double().cpu().numpy(), N.element_noise(SEED, SID, rows(n), D, 1, False)[:, 2])
    lim = 5 / n**0.5
    for a, b in ((fa, fb), (fa, z), (fb, z)):
        assert abs(float(torch.corrcoef(torch.stack([a.double(), b.double()]))[0, 1])) < lim


def test_independence_of_the_draws():
    n, D = 1 << 20, 4
    _, f, _, _ = sample("value_randn", n, D, True)
    f = f.double()
    assert not torch.equal(f[0::2], f[1::2])  # + and - rows of a direction differ
    assert abs(float(torch.corrcoef(torch.stack([f[0::2], f[1::2]]))[0, 1])) < 5 / (n / 2) ** 0.5
    _, g, _, _ = sample("value_randn", n, D, True, stream_id=SID + 1)  # the next generation
    assert abs(float(torch.corrcoef(torch.stack([f, g.double()]))[0, 1])) < 5 / n**0.5
    # the noise against the population's own z: x = mu + sigma z with mu = 0, sigma = 1
    z = torch.empty(n, 4, device=DEV)
    ops.sample_eval(ops.OBJ_NONE, z, torch.zeros(4, device=DEV), torch.ones(4, device=DEV), n_rows=n, symmetric=False, seed=SEED, stream_id=SID)
    _, h, _, _ = sample("value_randn", n, 4, False)
    for c in range(4):
        assert abs(float(torch.corrcoef(torch.stack([z[:, c].double(), h.double()]))[0, 1])) < 5 / n**0.5
    # two occurrences in one row are independent; both transforms have the stated distribution
    from scipy import stats

    _, t, _, _ = sample("two_uniforms", 200_000, 4, False)
    assert stats.kstest(t.cpu().numpy(), stats.triang(c=0.5, loc=0, scale=2).cdf).pvalue > 1e-3
    assert stats.kstest(f[:200_000].cpu().numpy(), "norm").pvalue > 1e-3


def test_eval_without_a_key_is_refused_and_leaves_f_untouched():
    o = obj("f7")
    X = torch.randn(32, 8, device=DEV)
    f = torch.full((32,), 7.0, device=DEV)
    rc = nat.lib().evok_eval(o.evok_objective_id, X.data_ptr(), 8, 32, 8, f.data_ptr(), nat.stream_of(X))
    torch.cuda.synchronize()
    assert rc == -9 and bool((f == 7.0).all())
    y = o(X)  # a direct call takes a fresh key
    assert y.shape == (32,) and bool(torch.isfinite(y).all())


# ------------------------------------------------------------------------------------------------ whole searchers
PAIR_GPU = _load("test_pair_objective_gpu.py")


@pytest.mark.parametrize("name", sorted(PAIR_GPU.SEARCHERS))
def test_graph_replay_and_lazy_bit_identical(name):
    o = obj("input_noise_sphere")
    D = 37 if name == "cmaes" else 130

    def run(lazy, graph):
        s = PAIR_GPU.SEARCHERS[name](PAIR_GPU._problem(o, D, lazy=lazy))
        if graph:
            s.enable_cuda_graph()
        hist = []
        for _ in range(6):
            s.step()
            hist.append([t.detach().clone() for t in PAIR_GPU._state(s)] + [s.population.evals.clone()])
        torch.cuda.synchronize()
        if graph:
            assert s._graph is not None
        return hist

    for group in PAIR_GPU.GROUPS[name]:
        ref = run(*group[0])
        assert not same(ref[0][-1], ref[1][-1])  # consecutive generations differ
        for lazy, graph in group[1:]:
            for g, (a, b) in enumerate(zip(ref, run(lazy, graph))):
                for x, y in zip(a, b):
                    assert same(x, y), (group[0], lazy, graph, g)


def test_checkpoint_resume_is_bit_identical(tmp_path):
    from evotorch_b200.algorithms import CMAES
    from evotorch_b200.logging import PicklingLogger

    o = obj("f7")

    def make():
        return CMAES(PAIR_GPU._problem(o, 150, lazy=False), stdev_init=1.0, popsize=200, separable=True)

    straight = make()
    straight.run(11)
    s = make()
    logger = PicklingLogger(s, interval=5, directory=str(tmp_path), prefix="nz", verbose=False, checkpoint=True)
    s.run(5)
    resumed = PicklingLogger.resume(logger.last_file_name)
    resumed.run(6)
    assert same(resumed.m, straight.m) and same(resumed.population.evals, straight.population.evals)
