"""FusedObjective with products, maxima, minima, running sums and conditionals, without a GPU: the language rules, the generated
source, byte-identical sources for the objectives of sums, the torch function against hand-written float64 formulas of the
classical test functions, pickling, and the NVRTC compilation of every kernel."""

import json
import math
import os
import pickle

import numpy as np
import pytest
import torch

from evotorch_b200 import jit
from evotorch_b200.objectives import FusedObjective

# the objectives of these tests, of tests/test_reduction_objective_gpu.py and of scripts/reduction_objective_bench.py
U_F12 = "where(x > 10, 100*(x - 10)**4, where(x < -10, 100*(-x - 10)**4, 0))"
U_F13 = "where(x > 5, 100*(x - 5)**4, where(x < -5, 100*(-x - 5)**4, 0))"
RED_SPECS = {
    "schwefel_2_22": dict(sums={"a": "abs(x)"}, prods={"p": "abs(x)"}, value="a + p"),
    "schwefel_1_2": dict(running={"c": "x"}, sums={"s": "c**2"}, value="s"),
    "schwefel_2_21": dict(maxs={"m": "abs(x)"}, value="m"),
    "griewank": dict(sums={"s": "x**2"}, prods={"p": "cos(x / sqrt(j + 1))"}, value="1 + s / 4000 - p"),
    "penalized_1": dict(sums={"b": "where(j == 0, 10*sin(pi*(1 + 0.25*(x + 1)))**2, 0) + where(j == D - 1, (0.25*(x + 1))**2, 0)",
                              "s": "(0.25*(x + 1))**2 * (1 + 10*sin(pi*(1 + 0.25*(xn + 1)))**2)", "u": U_F12},
                        value="pi / D * (b + s) + u"),
    "penalized_2": dict(sums={"b": "where(j == 0, sin(3*pi*x)**2, 0) + where(j == D - 1, (x - 1)**2 * (1 + sin(2*pi*x)**2), 0)",
                              "s": "(x - 1)**2 * (1 + sin(3*pi*xn)**2)", "u": U_F13},
                        value="0.1 * (b + s) + u"),
    # every kind in one accumulator: two running sums, a pair min, an element max of running sums, an element product, a pair sum
    "mixed": dict(running={"c": "x", "q": "abs(x) / D"}, sums={"s": "(xn - x)**2"}, mins={"lo": "x * xn"}, maxs={"hi": "c - q"},
                  prods={"p": "1 + 0.001 * q"}, value="s / D + hi - lo + p"),
    "pair_product_min": dict(prods={"p": "1 + 0.01 * (xn - x) / D"}, mins={"m": "-abs(x - xn)"}, value="p + m"),
    "penalty": dict(sums={"u": U_F12}, mins={"m": "where(j == D - 1, x, 0)"}, value="u + m"),
}


def make(name, **kw):
    spec = dict(RED_SPECS[name], **kw)
    return FusedObjective(name, spec.pop("sums", None), spec.pop("value"), spec.pop("data", None), **spec)


def spec_of(name):
    spec = dict(RED_SPECS[name])
    return jit.ObjectiveSpec(spec.pop("sums", None), spec.pop("value"), **spec)


# ------------------------------------------------------------------------------------------------ the language
@pytest.mark.parametrize("kw,match", [
    (dict(sums={"s": "c * xn"}, value="s", running={"c": "x"}), "'c' in a pair term; a running sum is usable in the element terms"),
    (dict(sums={"s": "c"}, value="s + c", running={"c": "x"}), "value: 'c' is a running sum; a running sum is usable in the element"),
    (dict(sums={"s": "c"}, value="s", running={"c": "x", "d": "c * x"}), r"running\['d'\]: 'c': a running term is an element term"),
    (dict(sums={"s": "c"}, value="s", running={"c": "s * x"}), r"running\['c'\]: 's': a running term"),
    (dict(sums={"s": "c"}, value="s", running={"c": "xn"}), "unknown name 'xn'"),
    (dict(sums={"s": "x < 1"}, value="s"), "Compare .* only as the condition of where"),
    (dict(sums={"s": "where(x, 1, 0)"}, value="s"), "condition of where must be one comparison"),
    (dict(sums={"s": "where(0 < x < 1, 1, 0)"}, value="s"), "condition of where must be one comparison"),
    (dict(sums={"s": "where(x < 1, 1)"}, value="s"), "where takes 3"),
    (dict(sums={"s": "where(x < 1, x > 0, 0)"}, value="s"), "Compare .* only as the condition"),
    (dict(sums={"s": "x"}, value="where(s > 0, s, 0) + (s > 1)"), "Compare"),
    (dict(sums={"a": "x", "b": "x"}, prods={"c": "x", "d": "x"}, maxs={"e": "x"}, value="a"), "1 to 4 reductions in all, got 5"),
    (dict(sums={}, prods={}, value="1"), "1 to 4 reductions in all, got 0"),
    (dict(sums={"s": "c + d + e"}, value="s", running={"c": "x", "d": "x", "e": "x"}), "at most 2"),
    (dict(sums={"s": "x"}, prods={"s": "x"}, value="s"), "'s' names two reductions"),
    (dict(sums={"s": "x"}, value="s", running={"s": "x"}), "'s' is also the name of a reduction"),
    (dict(maxs={"cos": "x"}, value="1"), "cannot name a max"),
    (dict(sums={"s": "c"}, value="s", running={"xn": "x"}), "cannot name a running sum"),
    (dict(sums={"s": "x"}, value=None), "needs a `value`"),
    (dict(sums={"s": "x"}, prods=["x"], value="s"), "prods: expected a dict"),
])
def test_rejected_expressions(kw, match):
    with pytest.raises(ValueError, match=match):
        jit.ObjectiveSpec(kw.pop("sums", None), kw.pop("value"), **kw)


def test_data_names_clash_with_reductions_and_running_sums():
    t = torch.randn(8)
    with pytest.raises(ValueError, match="'m' is the name of a max"):
        FusedObjective("clash", maxs={"m": "x"}, value="m", data={"m": t})
    with pytest.raises(ValueError, match="'c' is the name of a running sum"):
        FusedObjective("clash", sums={"s": "c"}, value="s", running={"c": "x"}, data={"c": t})
    with pytest.raises(ValueError, match="needs a `value`"):
        FusedObjective("no_value", sums={"s": "x"})


def test_running_terms_and_reductions_take_data():
    t, lam = torch.randn(6), torch.tensor([0.5])
    f = FusedObjective("shifted_schwefel_1_2", running={"c": "x - o"}, sums={"s": "c**2"}, maxs={"m": "lam * abs(x - o)"},
                       value="s + m", data={"o": t, "lam": lam})
    X = torch.randn(4, 6, dtype=torch.float64)
    z = X - t.double()
    want = (z.cumsum(-1) ** 2).sum(-1) + 0.5 * z.abs().amax(-1)
    torch.testing.assert_close(f(X), want, rtol=1e-12, atol=1e-12)
    src = f.source
    assert "void running(float x, int64_t j, const float (&d)[1], float (&h)[1])" in src
    assert "void add(float x, int64_t j, const float (&d)[1], const float (&r)[1])" in src


# ------------------------------------------------------------------------------------------------ the generated source
def _source(*body):
    return "\n".join(['#include "evok_sampler.cuh"', "", "namespace evok_user {", "struct Acc {", *body, "};", "}  // namespace evok_user", ""])


def test_generated_sources_spelt_out():
    ctor = "  __device__ __forceinline__ explicit Acc(int64_t D) : Df((float)D) {}"
    assert spec_of("griewank").source == _source(
        "  float Df;", "  float s0 = 0.f, s1 = 1.f;", ctor,
        "  __device__ __forceinline__ void add(float x, int64_t j) {", "    const float jf = (float)j;", "    s0 += (x * x);",
        "    s1 *= cosf((x / sqrtf((jf + 1.0f))));", "  }",
        "  __device__ __forceinline__ float finish(int64_t) {", "    const float S_s = evok::warp_sum(s0);",
        "    const float S_p = evok::warp_prod(s1);", "    return ((1.0f + (S_s / 4000.0f)) - S_p);", "  }")
    assert spec_of("schwefel_2_21").source == _source(
        "  float Df;", "  float s0 = -evok::inf();", ctor,
        "  __device__ __forceinline__ void add(float x, int64_t j) {", "    s0 = evok::max_nan(s0, fabsf(x));", "  }",
        "  __device__ __forceinline__ float finish(int64_t) {", "    const float S_m = evok::warp_max(s0);", "    return S_m;", "  }")
    assert jit.ObjectiveSpec(None, "m", mins={"m": "x * xn"}).source == _source(
        "  static constexpr bool kPairs = true;", "  float Df;", "  float s0 = evok::inf();", ctor,
        "  __device__ __forceinline__ void add(float x, int64_t j) {", "  }",
        "  __device__ __forceinline__ void add_pair(float x, float xn, int64_t j) {", "    s0 = evok::min_nan(s0, (x * xn));", "  }",
        "  __device__ __forceinline__ float finish(int64_t) {", "    const float S_m = evok::warp_min(s0);", "    return S_m;", "  }")
    assert spec_of("schwefel_1_2").source == _source(
        "  static constexpr bool kRunning = true;", "  static constexpr int kRunningSums = 1;", "  float Df;", "  float s0 = 0.f;", ctor,
        "  __device__ __forceinline__ void running(float x, int64_t j, float (&h)[1]) {", "    h[0] = x;", "  }",
        "  __device__ __forceinline__ void add(float x, int64_t j, const float (&r)[1]) {", "    s0 += (r[0] * r[0]);", "  }",
        "  __device__ __forceinline__ float finish(int64_t) {", "    const float S_s = evok::warp_sum(s0);", "    return S_s;", "  }")
    assert "((x > 10.0f) ? (100.0f * ((x - 10.0f) * (x - 10.0f) * (x - 10.0f) * (x - 10.0f))) : ((x < (-10.0f)) ?" in spec_of("penalized_1").source
    assert "((jf == 0.0f) ?" in spec_of("penalized_1").source


def test_sources_of_the_sum_language_are_unchanged():
    """Every objective of the existing CPU tests generates byte for byte the source it generated before products, maxima, minima,
    running sums and conditionals existed (tests/golden/objective_sources.json, recorded then); the source is the compile-cache key."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "objective_sources.json")
    with open(path) as fh:
        golden = json.load(fh)
    assert len(golden) >= 14
    for key, g in golden.items():
        spec = jit.ObjectiveSpec(g["sums"], g["value"], g["kinds"] or None)
        assert spec.source == g["source"], key
        kw = jit.ObjectiveSpec(g["sums"], g["value"], g["kinds"] or None, prods=None, maxs={}, mins=None, running={})
        assert kw.source == g["source"], key


# ------------------------------------------------------------------------------------------------ torch_fn in float64
def np_f2(X):
    return np.abs(X).sum(-1) + np.abs(X).prod(-1)


def np_f3(X):
    D = X.shape[-1]
    return sum(X[..., : j + 1].sum(-1) ** 2 for j in range(D))


def np_f4(X):
    return np.abs(X).max(-1)


def np_f11(X):
    j = np.arange(X.shape[-1])
    return 1 + (X**2).sum(-1) / 4000 - np.cos(X / np.sqrt(j + 1)).prod(-1)


def np_u(x, a, k, m):
    return np.where(x > a, k * (x - a) ** m, np.where(x < -a, k * (-x - a) ** m, 0.0))


def np_f12(X):
    D = X.shape[-1]
    y = 1 + (X + 1) / 4
    inner = (10 * np.sin(np.pi * y[..., 0]) ** 2 + ((y[..., :-1] - 1) ** 2 * (1 + 10 * np.sin(np.pi * y[..., 1:]) ** 2)).sum(-1)
             + (y[..., -1] - 1) ** 2)
    return np.pi / D * inner + np_u(X, 10, 100, 4).sum(-1)


def np_f13(X):
    inner = (np.sin(3 * np.pi * X[..., 0]) ** 2 + ((X[..., :-1] - 1) ** 2 * (1 + np.sin(3 * np.pi * X[..., 1:]) ** 2)).sum(-1)
             + (X[..., -1] - 1) ** 2 * (1 + np.sin(2 * np.pi * X[..., -1]) ** 2))
    return 0.1 * inner + np_u(X, 5, 100, 4).sum(-1)


FORMULAS = {"schwefel_2_22": np_f2, "schwefel_1_2": np_f3, "schwefel_2_21": np_f4, "griewank": np_f11, "penalized_1": np_f12,
            "penalized_2": np_f13}


@pytest.mark.parametrize("batch", [(), (3,), (2, 3)])
@pytest.mark.parametrize("D", [1, 2, 5, 33])
@pytest.mark.parametrize("name", sorted(FORMULAS))
def test_torch_fn_against_the_float64_formulas(name, D, batch):
    g = torch.Generator().manual_seed(D + len(batch))
    X = torch.rand(*batch, 7, D, generator=g, dtype=torch.float64) * 30 - 15  # both sides of the penalties' thresholds
    got = spec_of(name).torch_fn(X)
    assert got.dtype == torch.float64 and got.shape == X.shape[:-1]
    np.testing.assert_allclose(got.numpy(), FORMULAS[name](X.numpy()), rtol=1e-12, atol=1e-9)


def test_empty_reductions_and_non_finite_terms_in_torch_fn():
    X = torch.tensor([[2.0]], dtype=torch.float64)  # D = 1: every pair reduction is empty
    for kw, want in [(dict(sums={"s": "x * xn"}, value="s"), 0.0), (dict(prods={"p": "x * xn"}, value="p"), 1.0),
                     (dict(maxs={"m": "x * xn"}, value="m"), -math.inf), (dict(mins={"m": "x * xn"}, value="m"), math.inf)]:
        assert float(jit.ObjectiveSpec(kw.pop("sums", None), kw.pop("value"), **kw).torch_fn(X)[0]) == want
    X = torch.tensor([[1.0, math.nan, 3.0], [1.0, math.inf, 3.0], [-math.inf, 2.0, 0.5]], dtype=torch.float64)
    for kw in (dict(prods={"r": "x"}), dict(maxs={"r": "x"}), dict(mins={"r": "x"}), dict(running={"c": "x"}, sums={"r": "c"})):
        got = jit.ObjectiveSpec(kw.pop("sums", None), "r", **kw).torch_fn(X)
        assert math.isnan(got[0])  # NaN propagates through every kind
    assert jit.ObjectiveSpec(None, "r", maxs={"r": "x"}).torch_fn(X)[1:].tolist() == [math.inf, 2.0]
    assert jit.ObjectiveSpec(None, "r", mins={"r": "x"}).torch_fn(X)[1:].tolist() == [1.0, -math.inf]
    assert jit.ObjectiveSpec(None, "r", prods={"r": "x"}).torch_fn(X)[1:].tolist() == [math.inf, -math.inf]
    # where: a comparison with NaN is false, != true, as in CUDA
    w = jit.ObjectiveSpec({"a": "where(x < 2, 1, 0)", "b": "where(x != 2, 1, 0)"}, "a + 10 * b")
    assert w.torch_fn(torch.tensor([[math.nan], [1.0], [2.0]], dtype=torch.float64)).tolist() == [10.0, 11.0, 0.0]


def test_running_sums_broadcast_over_the_data_batch():
    o = torch.randn(3, 5)
    f = FusedObjective("shifted_schwefel_1_2", running={"c": "x - o"}, sums={"s": "c**2"}, value="s", data={"o": o})
    X = torch.randn(4, 5, dtype=torch.float64)
    got = f(X)
    assert got.shape == (3, 4)
    want = ((X[None] - o.double()[:, None]).cumsum(-1) ** 2).sum(-1)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ the object
def test_pickle_repr_and_with_data():
    f = make("mixed")
    g = pickle.loads(pickle.dumps(f))
    assert (g.sums, g.prods, g.maxs, g.mins, g.running, g.value) == (f.sums, f.prods, f.maxs, f.mins, f.running, f.value)
    assert g.source == f.source and g.evok_objective_id == f.evok_objective_id
    X = torch.randn(3, 9, dtype=torch.float64)
    assert torch.equal(g(X), f(X))
    assert repr(make("schwefel_2_21")) == "FusedObjective('schwefel_2_21', sums={}, value='m', maxs={'m': 'abs(x)'})"
    t = torch.randn(6)
    h = FusedObjective("shifted_griewank", sums={"s": "(x - o)**2"}, prods={"p": "cos((x - o) / sqrt(j + 1))"}, value="1 + s / 4000 - p",
                       data={"o": t})
    k = h.with_data(o=t + 1)
    assert k.prods == h.prods and k.source == h.source
    Y = torch.randn(2, 6)
    torch.testing.assert_close(k(Y), h(Y - 1))
    assert torch.equal(pickle.loads(pickle.dumps(h))(Y), h(Y))
    assert "prods={'p': " in repr(h) and "data={'o': (6,)}" in repr(h)


# ------------------------------------------------------------------------------------------------ NVRTC, no GPU needed
# (sinf / cosf of a large argument take libdevice's slow path, whose local array ptxas counts as a spill in some kernels, with or
# without the new reductions: the penalized functions are left out here for that reason)
@pytest.mark.parametrize("name", ["griewank", "schwefel_1_2", "schwefel_2_21", "mixed", "pair_product_min", "penalty"])
def test_every_kernel_compiles_for_sm_90a_without_spills(name):
    f = make(name)
    f.compile_batched()
    assert len(f.kernel_info) == jit.N_KERNELS and len(f.batched_kernel_info) == jit.N_BATCHED_KERNELS
    for info in (f.kernel_info, f.batched_kernel_info):
        for kernel, i in info.items():
            assert i["spill_stores"] == 0 and i["spill_loads"] == 0 and i["registers"] <= 80, (name, kernel, i)
    print(name, "registers", sorted({i["registers"] for i in f.kernel_info.values()}), sorted({i["registers"] for i in f.batched_kernel_info.values()}))


def test_running_sums_with_data_compile_without_spills():
    t = torch.randn(8)
    f = FusedObjective("shifted_schwefel_1_2", running={"c": "x - o", "q": "w * x"}, sums={"s": "c**2 + q"}, value="s",
                       data={"o": t, "w": t})
    f.compile_batched()
    for info in (f.kernel_info, f.batched_kernel_info):
        for kernel, i in info.items():
            assert i["spill_stores"] == 0 and i["spill_loads"] == 0, (kernel, i)
