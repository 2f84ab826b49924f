"""FusedObjective with data, without a GPU: the language rules, the generated source, the compile cache, the torch function against
hand-written numpy formulas in float64, pickling, and the Python fallbacks of the batched functional API."""

import importlib.util
import os
import pickle

import numpy as np
import pytest
import torch

from evotorch_b200 import jit
from evotorch_b200.algorithms.functional import cem, cem_ask, cem_ask_and_evaluate, cem_tell, pgpe, pgpe_ask, pgpe_ask_and_evaluate, pgpe_tell
from evotorch_b200.objectives import FusedObjective

LSQ = ({"s": "w * (x - t)**2"}, "s + lam * D")
SHIFTED_RASTRIGIN = ({"s": "(x - o)**2 - 10 * cos(2 * pi * (x - o))"}, "10 * D + s")
SHIFTED_ROSENBROCK = ({"s": "100*((xn - o_n) - (x - o)**2)**2 + (1 - (x - o))**2"}, "s")
SHIFTED_SPHERE = ({"s": "(x - o)**2"}, "s")


def _load(filename):
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), filename)
    spec = importlib.util.spec_from_file_location("_" + filename[:-3], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed + sum(shape)))


# ------------------------------------------------------------------------------------------------ the language
def test_accepted_expressions():
    t, lam = rnd(8), torch.tensor([0.5])
    for sums, value, data in [(LSQ[0], LSQ[1], {"t": t, "w": t.abs(), "lam": lam}),
                              (SHIFTED_ROSENBROCK[0], "s", {"o": t}),
                              ({"s": "x * xn * lam + o * o_n", "a": "abs(x - o) * j"}, "s + a / lam", {"o": t, "lam": lam}),
                              ({"s": "x * lam"}, "s", {"lam": torch.full((3, 1), 2.0)}),
                              ({"s": "x"}, "s", {"a": t, "b": t, "c": t, "d": t})]:
        spec = jit.ObjectiveSpec(sums, value, jit.data_kinds(data))
        assert "kData" in spec.source and f"kVectors = {sum(v.shape[-1] != 1 for v in data.values())}" in spec.source


@pytest.mark.parametrize("sums,value,data,match", [
    ({"s": "x"}, "s", {"x": "vec"}, "cannot name data"),
    ({"s": "x"}, "s", {"xn": "vec"}, "cannot name data"),
    ({"s": "x"}, "s", {"pi": "vec"}, "cannot name data"),
    ({"s": "x"}, "s", {"cos": "vec"}, "cannot name data"),
    ({"s": "x"}, "s", {"t_n": "vec"}, "does not end in '_n'"),
    ({"s": "x"}, "s", {"2t": "vec"}, "cannot name data"),
    ({"s": "x"}, "s", {"s": "vec"}, "is the name of a sum"),
    ({"s": "x * t_n"}, "s", {"t": "vec"}, "only a pair term"),
    ({"s": "x * xn * lam_n"}, "s", {"lam": "scalar"}, "is a scalar"),
    ({"s": "x"}, "s * lam_n", {"lam": "scalar"}, "is a scalar"),
    ({"s": "x"}, "s + t", {"t": "vec"}, "in the terms of `sums` only"),
    ({"s": "x * xn"}, "s + t_n", {"t": "vec"}, "in the terms of `sums` only"),
    ({"s": "x * u"}, "s", {"t": "vec"}, "unknown name 'u'"),
    ({"s": "x"}, "s", {"a": "vec", "b": "vec", "c": "vec", "d": "vec", "f": "vec"}, "at most 4"),
    ({"s": "x"}, "s", {"t": "double"}, "float32"),
    ({"s": "x"}, "s", {"t": "int"}, "float32"),
    ({"s": "x"}, "s", {"t": "zero_dim"}, "at least one dimension"),
    ({"s": "x"}, "s", {"t": "list"}, "float32"),
])
def test_rejected_expressions(sums, value, data, match):
    made = {"vec": rnd(8), "scalar": torch.tensor([1.0]), "double": rnd(8).double(), "int": torch.arange(8), "zero_dim": torch.tensor(1.0),
            "list": [1.0, 2.0]}
    with pytest.raises(ValueError, match=match):
        FusedObjective("rejected", sums, value, {n: made[k] for n, k in data.items()})


def test_wrong_vector_length_at_call_time():
    f = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": rnd(8)})
    with pytest.raises(ValueError, match="length 8, the rows have length 9"):
        f(torch.zeros(3, 9))
    with pytest.raises(ValueError, match="one batch shape"):
        FusedObjective("two_batches", {"s": "(x - o) * w"}, "s", {"o": rnd(3, 8), "w": rnd(4, 8)})
    with pytest.raises(ValueError, match="expected the data names"):
        f.with_data(t=rnd(8))


def test_no_data_sources_are_unchanged():
    """The source of an objective without data does not depend on the data language: every no-data objective of the existing
    tests generates the same text with data=None, data={} and through FusedObjective, with no data code in it."""
    specs = dict(_load("test_pair_objective.py").PAIR_SPECS)
    specs.update(getattr(_load("test_fused_objective.py"), "SPECS", {}))
    assert len(specs) >= 4
    for name, (sums, value) in specs.items():
        plain = jit.ObjectiveSpec(sums, value).source
        assert jit.ObjectiveSpec(sums, value, {}).source == plain, name
        assert jit.ObjectiveSpec(sums, value, jit.data_kinds({})).source == plain, name
        assert "kData" not in plain and "DataBinding" not in plain and "vec[" not in plain, name
    # the text of the element-only and pair languages, spelt out for one objective of each
    assert jit.ObjectiveSpec({"s": "x**2"}, "s").source == "\n".join([
        '#include "evok_sampler.cuh"', "", "namespace evok_user {", "struct Acc {", "  float Df;", "  float s0 = 0.f;",
        "  __device__ __forceinline__ explicit Acc(int64_t D) : Df((float)D) {}",
        "  __device__ __forceinline__ void add(float x, int64_t j) {", "    s0 += (x * x);", "  }",
        "  __device__ __forceinline__ float finish(int64_t) {", "    const float S_s = evok::warp_sum(s0);", "    return S_s;", "  }", "};",
        "}  // namespace evok_user", ""])


def test_same_expressions_and_kinds_compile_once():
    a = FusedObjective("lsq", *LSQ, data={"t": rnd(8), "w": rnd(8).abs(), "lam": torch.tensor([0.1])})
    n = len(jit._cache)
    b = FusedObjective("lsq", *LSQ, data={"t": rnd(12), "w": rnd(12).abs(), "lam": torch.tensor([0.7])})
    c = a.with_data(t=rnd(5, 8), w=rnd(8).abs(), lam=torch.ones(5, 1))
    assert len(jit._cache) == n and a.source == b.source == c.source and a.kernel_info is b.kernel_info
    # another kind is another source: lam as a vector
    d = FusedObjective("lsq", {"s": "w * (x - t)**2 + lam"}, "s", data={"t": rnd(8), "w": rnd(8), "lam": rnd(8)})
    assert d.source != a.source


def test_documented_objectives_do_not_spill():
    o = rnd(8)
    for sums, value, data in [(LSQ[0], LSQ[1], {"t": o, "w": o, "lam": torch.ones(1)}), (*SHIFTED_SPHERE, {"o": o}),
                              (*SHIFTED_RASTRIGIN, {"o": o}), (*SHIFTED_ROSENBROCK, {"o": o})]:
        f = FusedObjective("documented", sums, value, data)
        f.compile_batched()
        assert len(f.kernel_info) == jit.N_KERNELS and len(f.batched_kernel_info) == jit.N_BATCHED_KERNELS
        for info in (f.kernel_info, f.batched_kernel_info):
            for kernel, i in info.items():
                assert i["spill_stores"] == 0 and i["spill_loads"] == 0 and i["registers"] <= 80, (sums, kernel, i)


# ------------------------------------------------------------------------------------------------ torch_fn in float64
def np_lsq(X, t, w, lam):
    return (w[..., None, :] * (X - t[..., None, :]) ** 2).sum(-1) + lam * X.shape[-1]


def np_shifted_rastrigin(X, o):
    z = X - o[..., None, :]
    return 10 * X.shape[-1] + (z**2 - 10 * np.cos(2 * np.pi * z)).sum(-1)


def np_shifted_rosenbrock(X, o):
    z = X - o[..., None, :]
    return (100 * (z[..., 1:] - z[..., :-1] ** 2) ** 2 + (1 - z[..., :-1]) ** 2).sum(-1)


@pytest.mark.parametrize("batch", [(), (3,), (2, 3)])
@pytest.mark.parametrize("D", [1, 2, 5, 33])
def test_torch_fn_against_numpy_in_float64(D, batch):
    X = rnd(*batch, 7, D, seed=1).double()
    o, w, lam = rnd(*batch, D, seed=2), rnd(*batch, D, seed=3).abs(), rnd(*batch, 1, seed=4)
    o64, w64, lam64 = (t.double().numpy() for t in (o, w, lam))
    # D = 1: a tensor with last dimension 1 is a scalar, which an element term takes as it takes a vector
    got = FusedObjective("lsq", *LSQ, data={"t": o, "w": w, "lam": lam})(X)
    np.testing.assert_allclose(got.numpy(), np_lsq(X.numpy(), o64, w64, lam64), rtol=1e-12, atol=1e-12)
    got = FusedObjective("shifted_rastrigin", *SHIFTED_RASTRIGIN, data={"o": o})(X)
    np.testing.assert_allclose(got.numpy(), np_shifted_rastrigin(X.numpy(), o64), rtol=1e-12, atol=1e-10)
    if D > 1:
        got = FusedObjective("shifted_rosenbrock", *SHIFTED_ROSENBROCK, data={"o": o})(X)
        assert got.dtype == torch.float64 and got.shape == X.shape[:-1]
        np.testing.assert_allclose(got.numpy(), np_shifted_rosenbrock(X.numpy(), o64), rtol=1e-12, atol=1e-12)
    else:
        with pytest.raises(ValueError, match="is a scalar"):
            FusedObjective("shifted_rosenbrock", *SHIFTED_ROSENBROCK, data={"o": o})


def test_torch_fn_broadcasts_the_data_batch_and_takes_one_solution():
    o = rnd(4, 6)
    f = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": o})
    X = rnd(5, 6, seed=9)
    got = f(X)  # an unbatched population against 4 data sets
    assert got.shape == (4, 5)
    np.testing.assert_allclose(got.numpy(), ((X[None] - o[:, None]) ** 2).sum(-1).numpy(), rtol=1e-6)
    one = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": o[0]})
    assert one(X[0]).shape == () and float(one(X[0])) == pytest.approx(float(((X[0] - o[0]) ** 2).sum()), rel=1e-6)


# ------------------------------------------------------------------------------------------------ the object
def test_pickle_with_data_and_repr():
    t, w, lam = rnd(8), rnd(8).abs(), torch.tensor([0.25])
    f = FusedObjective("lsq", *LSQ, data={"t": t, "w": w, "lam": lam})
    g = pickle.loads(pickle.dumps(f))
    X = rnd(3, 8, seed=5)
    assert list(g.data) == ["t", "w", "lam"] and all(torch.equal(g.data[n], f.data[n]) for n in f.data)
    assert torch.equal(g(X), f(X)) and g.source == f.source
    assert repr(f) == ("FusedObjective('lsq', sums={'s': 'w * (x - t)**2'}, value='s + lam * D', "
                       "data={'t': (8,), 'w': (8,), 'lam': (1,)})")
    plain = FusedObjective("plain_sphere", {"s": "x**2"}, "s")
    assert plain.data == {} and repr(plain) == "FusedObjective('plain_sphere', sums={'s': 'x**2'}, value='s')"
    assert pickle.loads(pickle.dumps(plain)).source == plain.source
    # the tensors are held by reference: a copy_ into them is what the next call evaluates
    h = f.with_data(t=t.clone(), w=w, lam=lam)
    before = h(X)
    h.data["t"].copy_(t + 1)
    assert not torch.equal(h(X), before) and torch.equal(h(X), f.with_data(t=t + 1, w=w, lam=lam)(X))


# ------------------------------------------------------------------------------------------------ the functional fallbacks
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_functional_fallbacks_with_per_item_data(dtype):
    B, D, n = 5, 6, 8
    targets = rnd(B, D, seed=11)
    f = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": targets})
    expr = lambda X: ((X - targets.to(dtype)[:, None, :]) ** 2).sum(-1)  # noqa: E731
    for center in (torch.zeros(B, D, dtype=dtype), torch.zeros(D, dtype=dtype)):  # a batched state, and one broadcast to the data
        st = pgpe(center_init=center, center_learning_rate=0.2, stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0)
        torch.manual_seed(3)
        values, evals = pgpe_ask_and_evaluate(st, popsize=n, objective=f)
        torch.manual_seed(3)
        asked = pgpe_ask(st, popsize=n)
        assert values.shape == (B, n, D) and evals.shape == (B, n) and evals.dtype == dtype
        assert torch.equal(values, asked.expand(B, n, D))
        torch.testing.assert_close(evals, expr(asked), rtol=1e-5, atol=1e-5)
        assert pgpe_tell(st, values, evals).stdev.shape == (B, D)
        cs = cem(center_init=center, parenthood_ratio=0.5, objective_sense="min", stdev_init=1.0)
        torch.manual_seed(4)
        values, evals = cem_ask_and_evaluate(cs, popsize=n, objective=f)
        torch.manual_seed(4)
        asked = cem_ask(cs, popsize=n)
        assert values.shape == (B, n, D) and torch.equal(values, asked.expand(B, n, D))
        torch.testing.assert_close(evals, expr(asked), rtol=1e-5, atol=1e-5)
        assert cem_tell(cs, values, evals).center.shape == (B, D)
    st = pgpe(center_init=torch.zeros(3, D), center_learning_rate=0.2, stdev_learning_rate=0.1, objective_sense="min", stdev_init=1.0)
    with pytest.raises(ValueError, match=r"\(3,\).*\(5,\)"):
        pgpe_ask_and_evaluate(st, popsize=n, objective=f)
