"""FusedObjective with noise (rand() / randn()) without a GPU: the language rules and messages, the generated sources, the
numpy restatement of the noise counters, the distribution of the torch function's noise, pickling, and the NVRTC compilation
of every kernel of the test objectives with no spills."""

import ctypes
import json
import math
import os
import pickle

import numpy as np
import pytest
import torch
from scipy import stats

from evotorch_b200 import _native as nat
from evotorch_b200 import jit
from oracle import es_oracle as O
from oracle import noise_oracle as N

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "noisy_objective_sources.json")

# the objectives of the tests (also of tests/test_noisy_objective_gpu.py and scripts/noisy_objective_bench.py)
NOISY_SPECS = {
    "value_rand": dict(sums={"s": "x"}, value="rand()"),
    "value_randn": dict(sums={"s": "x"}, value="randn()"),
    "elem_rand": dict(sums={"s": "rand()"}, value="s"),
    "elem_rand_j": dict(sums={"s": "(j + 1) * rand()"}, value="s"),
    "elem_randn": dict(sums={"s": "(x + randn())**2"}, value="s"),
    "f7": dict(sums={"s": "(j + 1) * x**4"}, value="s + rand()"),
    "bbob_rastrigin": dict(sums={"s": "x**2 - 10 * cos(2 * pi * x)"}, value="(10 * D + s) * exp(0.01 * randn())"),
    "input_noise_sphere": dict(sums={"s": "(x + 0.1 * randn())**2"}, value="s"),
    "two_uniforms": dict(sums={"s": "x"}, value="rand() + rand()"),
    "where_noise": dict(sums={"s": "where(rand() < 0.25, x**2, randn())"}, maxs={"m": "abs(x) + rand()"}, value="s + m"),
    "running_pair_noise": dict(running={"c": "x"}, sums={"s": "c * randn()", "p": "(xn - x)**2"}, value="s + p + randn()"),
}


def spec(name):
    kw = dict(NOISY_SPECS[name])
    return jit.ObjectiveSpec(kw.pop("sums", None), kw.pop("value"), **kw)


def make(name):
    from evotorch_b200.objectives import FusedObjective

    return FusedObjective("noisy_" + name, **NOISY_SPECS[name])


# ------------------------------------------------------------------------------------------------ language
@pytest.mark.parametrize("name", sorted(NOISY_SPECS))
def test_noise_is_accepted_where_allowed(name):
    sp = spec(name)
    assert sp.noisy
    assert "static constexpr bool kNoise = true;" in sp.source


def test_element_and_value_occurrences_are_numbered_in_source_order():
    sp = jit.ObjectiveSpec({"s": "rand() + randn()", "t": "where(x < 0, randn(), rand())"}, "s + t + randn() + rand()")
    assert sp.element_draws.normal == [False, True, True, False] and sp.value_draws.normal == [True, False]
    assert "static constexpr int kDraws = 4;" in sp.source and "kNormalDraws = 6u;" in sp.source
    assert "evok::value_randn(key, sw, row, 4)" in sp.source and "evok::value_rand(key, sw, row, 5)" in sp.source
    # after the data vectors: the draws are the column entries d[kVectors + k]
    sp = jit.ObjectiveSpec({"s": "w * (x - t + randn())**2"}, "s", {"t": True, "w": True, "lam": False})
    assert "const float (&d)[3]" in sp.source and "d[2]" in sp.source


def test_an_objective_without_noise_is_not_noisy():
    for sums, value in (({"s": "x**2"}, "s"), ({"s": "100*(xn - x**2)**2"}, "s"), ({"rand_s": "x"}, "rand_s")):
        sp = jit.ObjectiveSpec(sums, value)
        assert not sp.noisy and "kNoise" not in sp.source and "PhiloxKey" not in sp.source


@pytest.mark.parametrize("kwargs,message", [
    (dict(sums={"s": "(xn - x) * randn()"}, value="s"), r"sums\['s'\]: randn\(\) draws noise, which is allowed in the element terms"),
    (dict(prods={"p": "xn + rand()"}, value="p"), r"prods\['p'\]: rand\(\) draws noise.*not in a pair term or a running term"),
    (dict(running={"c": "x + randn()"}, sums={"s": "c"}, value="s"), r"running\['c'\]: randn\(\) draws noise"),
    (dict(sums={"s": "rand(2)"}, value="s"), r"sums\['s'\]: rand\(\) takes no arguments, got 'rand\(2\)'"),
    (dict(sums={"s": "x"}, value="s + randn(s)"), r"value: randn\(\) takes no arguments"),
    (dict(sums={"s": "randn(scale=2)"}, value="s"), r"takes no arguments"),
    (dict(sums={"s": "rand() + rand() + rand()", "t": "randn() + randn()"}, value="s + t"),
     r"sums\['t'\]: at most 4 occurrences of rand\(\) / randn\(\) in the element terms"),
    (dict(sums={"s": "x"}, value="s + rand() + rand() + randn() + randn() + rand()"), r"value: at most 4 occurrences .* in `value`"),
])
def test_noise_is_refused_elsewhere(kwargs, message):
    kw = dict(kwargs)
    with pytest.raises(ValueError, match=message):
        jit.ObjectiveSpec(kw.pop("sums", None), kw.pop("value"), **kw)


def test_rand_and_randn_stay_usable_as_names():
    """Only a call draws: `rand` and `randn` still name a reduction, a running sum or data, as before noise."""
    sp = jit.ObjectiveSpec({"rand": "x**2"}, "rand + randn()")
    assert "S_rand" in sp.source and sp.value_draws.normal == [True] and not sp.element_draws.normal
    sp = jit.ObjectiveSpec({"s": "randn * rand()"}, "s", running={"randn": "x"})
    assert sp.element_draws.normal == [False]
    assert jit.data_kinds({"randn": torch.zeros(3)}) == {"randn": True}
    X = torch.randn(5, 4, dtype=torch.float64)
    assert torch.allclose(jit.ObjectiveSpec({"rand": "x**2"}, "rand").torch_fn(X), (X**2).sum(-1))


def test_generated_sources_are_pinned():
    golden = json.load(open(GOLDEN))
    assert sorted(golden) == sorted(NOISY_SPECS)
    for name in NOISY_SPECS:
        assert spec(name).source == golden[name], name


# ------------------------------------------------------------------------------------------------ counters
def test_noise_counters_are_philox_of_the_stated_counter():
    seed, sid = 0x0123_4567_89AB_CDEF, (5 << 32) | 77
    rows = np.array([0, 1, 2, 3, 1000, 2**32 + 5, 2**40 + 3], dtype=np.uint64)
    for k, normal in ((0, False), (3, True)):
        got = N.element_noise(seed, sid, rows, 11, k, normal)
        for i, r in enumerate(rows):
            for j in range(11):
                c = (j // 4, int(r) & 0xFFFFFFFF, 0x80000000 | (k << 24) | ((int(r) >> 32) & 0xFFFFFF), sid & 0xFFFFFFFF)
                w = O.philox4x32_10(*[np.array([v], dtype=np.uint32) for v in c], seed & 0xFFFFFFFF, ((seed >> 32) ^ (sid >> 32)) & 0xFFFFFFFF)
                if normal:
                    a, b = O._box_muller(w[0], w[1]) if j % 4 < 2 else O._box_muller(w[2], w[3])
                    want = (a if j % 2 == 0 else b)[0]
                else:
                    want = float(w[j % 4][0] >> 8) * 2.0**-24
                assert got[i, j] == want
    v = N.value_noise(seed, sid, rows, 4, False)
    w = O.philox4x32_10(*N.noise_counter(0xFFFFFFFF, rows, 4, sid), seed & 0xFFFFFFFF, ((seed >> 32) ^ (sid >> 32)) & 0xFFFFFFFF)
    assert np.array_equal(v, (w[0] >> 8).astype(np.float64) * 2.0**-24)


def test_uniforms_are_exact_float32_in_the_unit_interval():
    w = np.array([0, 255, 256, 2**31, 2**32 - 1], dtype=np.uint32)
    u = N.uniform24(w)
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)
    assert u[0] == 0.0 and u[1] == 0.0 and u[-1] == 1.0 - 2.0**-24


def test_no_noise_counter_equals_a_sample_counter():
    """Exhaustively over small ranges and at the 32-bit row boundaries: every noise counter of rows, groups, occurrences and
    the value word against every sample counter of the same units and groups."""
    sw = 3
    units = np.concatenate([np.arange(0, 64), np.arange(2**32 - 8, 2**32 + 8), [2**48, 2**56 - 1]]).astype(np.uint64)
    q = np.arange(0, 40, dtype=np.uint64)
    Q, Uu = np.meshgrid(q, units, indexing="ij")
    samples = set(zip(*(c.ravel().tolist() for c in N.sample_counter(Q, Uu, sw))))
    noise = set()
    for k in range(8):
        for x in (Q, np.full_like(Q, N.VALUE_X)):
            noise |= set(zip(*(c.ravel().tolist() for c in N.noise_counter(x, Uu, k, sw))))
    assert len(noise) == 8 * 2 * Q.size - 8 * (len(q) - 1) * len(units)  # the value word repeats over q: one per (k, row)
    assert not samples & noise


# ------------------------------------------------------------------------------------------------ the torch function
def _ks(sample, cdf):
    return stats.kstest(sample.double().numpy().ravel(), cdf).pvalue


def test_torch_function_draws_the_stated_distributions():
    torch.manual_seed(0)
    X = torch.zeros(20_000, 3)
    assert _ks(spec("value_rand").torch_fn(X), "uniform") > 1e-3
    assert _ks(spec("value_randn").torch_fn(X), "norm") > 1e-3
    # sums {"s": "rand()"} at D = 3: the sum of 3 independent uniforms per row (Irwin-Hall)
    irwin_hall = lambda t: np.clip(np.where(t < 1, t**3 / 6, np.where(t < 2, (-2 * t**3 + 9 * t**2 - 9 * t + 3) / 6,  # noqa: E731
                                                                     1 - (3 - t)**3 / 6)), 0, 1)
    assert _ks(spec("elem_rand").torch_fn(X), irwin_hall) > 1e-3
    # two occurrences are two independent draws: rand() + rand() is triangular on [0, 2], not 2 * rand()
    tri = stats.triang(c=0.5, loc=0, scale=2).cdf
    s = spec("two_uniforms").torch_fn(torch.zeros(20_000, 1))
    assert _ks(s, tri) > 1e-3 and _ks(s / 2, "uniform") < 1e-6


def test_torch_function_noise_is_per_row_and_column_in_float64_and_batches():
    torch.manual_seed(1)
    X = torch.zeros(2, 5000, 4, dtype=torch.float64)
    f = spec("elem_randn").torch_fn(X)  # sum_j (0 + z_j)^2: chi-square with 4 degrees of freedom
    assert f.shape == (2, 5000) and f.dtype == torch.float64
    assert _ks(f, stats.chi2(4).cdf) > 1e-3
    f = spec("input_noise_sphere").torch_fn(torch.ones(4000, 6))
    assert abs(float(f.mean()) - 6 * (1 + 0.01)) < 0.1


# ------------------------------------------------------------------------------------------------ pickling and compilation
def test_noisy_objective_pickles_as_its_expressions():
    o = make("where_noise")
    assert o.noisy
    p = pickle.loads(pickle.dumps(o))
    assert p.noisy and p.source == o.source and p.evok_objective_id == o.evok_objective_id
    assert not make_plain().noisy


def make_plain():
    from evotorch_b200.objectives import FusedObjective

    return FusedObjective("plain_sphere_for_noise_tests", sums={"s": "x**2"}, value="s")


def test_eval_without_a_key_refuses_a_noisy_objective_and_launches_nothing():
    o = make("f7")
    lib = nat.lib()
    before = lib.evok_launch_count()
    buf = (ctypes.c_float * 16)()
    rc = lib.evok_eval(o.evok_objective_id, ctypes.addressof(buf), 4, 4, 4, ctypes.addressof(buf), None)
    assert rc == -9 and b"noise" in lib.evok_error_string(rc)
    assert lib.evok_launch_count() == before
    assert lib.evok_objective_declare_noise(0) == -3  # only a registered id declares noise


@pytest.mark.parametrize("name", sorted(NOISY_SPECS))
def test_every_kernel_compiles_without_spills(name):
    sp = spec(name)
    for exprs in (None, jit.batched_kernel_expressions()):
        c = jit.compile_source(sp.source, exprs)
        for e, info in c.kernel_info.items():
            assert info["spill_stores"] == 0 and info["spill_loads"] == 0, (name, e, info)
