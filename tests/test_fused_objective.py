"""FusedObjective without a GPU: the expression translator, the NVRTC compilation for sm_90a and the registration ABI."""

import ctypes
import math
import pickle
import time

import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200 import jit

E_NULLPTR, E_BADSIZE, E_BADENUM = -1, -2, -3  # EVOK_E_* of include/evok.h
USER_BASE, USER_CAPACITY, N_KERNELS = 64, 256, 22

# the objectives of the tests (and of scripts/fused_objective_bench.py), with a hand-written float64 formula each
SPECS = {
    "sphere_twin": ({"s": "x**2"}, "s"),
    "styblinski_tang": ({"s": "x**4 - 16*x**2 + 5*x"}, "0.5 * s"),
    "ellipsoid": ({"s": "1e6 ** (j / (D - 1)) * x**2"}, "s"),
    "rastrigin_twin": ({"a": "x**2", "c": "cos(2*pi*x)"}, "10*D + a - 10*c"),
    "ackley_twin": ({"a": "x**2", "c": "cos(2*pi*x)"}, "-20*exp(-0.2*sqrt(a/D)) - exp(c/D) + 20 + e"),
    "schwefel": ({"s": "x * sin(sqrt(abs(x)))"}, "418.9829 * D - s"),
}


def f64(name: str, X: torch.Tensor) -> torch.Tensor:
    X = X.double()
    D = X.shape[-1]
    j = torch.arange(D, dtype=torch.float64)
    if name == "sphere_twin":
        return (X**2).sum(-1)
    if name == "styblinski_tang":
        return 0.5 * (X**4 - 16 * X**2 + 5 * X).sum(-1)
    if name == "ellipsoid":
        return (1e6 ** (j / (D - 1)) * X**2).sum(-1)
    if name == "rastrigin_twin":
        return 10 * D + (X**2 - 10 * torch.cos(2 * math.pi * X)).sum(-1)
    if name == "ackley_twin":
        return (-20 * torch.exp(-0.2 * torch.sqrt((X**2).mean(-1))) - torch.exp(torch.cos(2 * math.pi * X).mean(-1)) + 20 + math.e)
    return 418.9829 * D - (X * torch.sin(torch.sqrt(X.abs()))).sum(-1)


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


# ------------------------------------------------------------------------------------------------ the translator
ACCEPTED_TERMS = ["x", "-x", "+x", "x + j - D", "x * 2.5 / D", "x**3", "x**-2", "x**0", "x**2.0", "x**0.5", "2**x", "x**(j/D)", "abs(x)",
                  "sqrt(abs(x))", "exp(-x)", "log(1 + x*x)", "sin(x)", "cos(2*pi*x)", "tan(x)", "tanh(x)", "floor(x)", "minimum(x, 1)",
                  "maximum(x, -e)", "1e-3 * x", "3"]


@pytest.mark.parametrize("term", ACCEPTED_TERMS)
def test_whitelisted_constructs_are_accepted(term):
    spec = jit.ObjectiveSpec({"s": term}, "s / D + 1")
    X = torch.linspace(0.25, 2.0, 21, dtype=torch.float64).reshape(3, 7)
    env = {"x": X, "j": torch.arange(7.0, dtype=torch.float64), "D": 7.0, "pi": math.pi, "e": math.e, "abs": abs, "sqrt": torch.sqrt,
           "exp": torch.exp, "log": torch.log, "sin": torch.sin, "cos": torch.cos, "tan": torch.tan, "tanh": torch.tanh,
           "floor": torch.floor, "minimum": lambda a, b: torch.fmin(a, torch.as_tensor(b, dtype=torch.float64)),
           "maximum": lambda a, b: torch.fmax(a, torch.as_tensor(b, dtype=torch.float64))}
    t = eval(term, {"__builtins__": {}}, env)  # noqa: S307 -- the test's own expressions
    want = torch.broadcast_to(torch.as_tensor(t, dtype=torch.float64), X.shape).sum(-1) / 7 + 1
    torch.testing.assert_close(spec.torch_fn(X), want, rtol=1e-12, atol=1e-12)
    assert "struct Acc" in spec.source


REJECTED = [
    ({"s": "x % 2"}, "s", "Mod"),
    ({"s": "x // 2"}, "s", "FloorDiv"),
    ({"s": "x if x else 0"}, "s", "IfExp"),
    ({"s": "x < 1"}, "s", "Compare"),
    ({"s": "y"}, "s", "unknown name 'y'"),
    ({"s": "s"}, "s", "unknown name 's'"),
    ({"s": "x"}, "s + x", "unknown name 'x'"),
    ({"s": "x"}, "s + j", "unknown name 'j'"),
    ({"s": "torch.sin(x)"}, "s", "not supported"),
    ({"s": "sinh(x)"}, "s", "'sinh' is not supported"),
    ({"s": "max(x, 1)"}, "s", "'max' is not supported"),
    ({"s": "minimum(x)"}, "s", "takes 2 argument"),
    ({"s": "sqrt(x=x)"}, "s", "keyword"),
    ({"s": "'x'"}, "s", "not a number"),
    ({"s": "1e39 * x"}, "s", "not a finite float32"),
    ({"s": "x +"}, "s", "not a Python expression"),
    ({"s": "x.real"}, "s", "Attribute"),
    ({"s": "[x]"}, "s", "List"),
    ({"s": "(lambda: x)()"}, "s", "not supported"),
    ({"s": "~x"}, "s", "Invert"),
    ({}, "1", "1 to 4"),
    ({"a": "x", "b": "x", "c": "x", "d": "x", "f": "x"}, "a", "1 to 4"),
    ({"x": "x"}, "x", "cannot name a sum"),
    ({"cos": "x"}, "cos", "cannot name a sum"),
    ({"s": "x"}, 3, "expected an expression string"),
]


@pytest.mark.parametrize("sums,value,message", REJECTED)
def test_rejected_constructs_name_what_is_allowed(sums, value, message):
    with pytest.raises(ValueError, match=message) as info:
        jit.ObjectiveSpec(sums, value)
    if "not supported" in str(info.value) or "unknown name" in str(info.value):
        assert "allowed:" in str(info.value) and "minimum" in str(info.value)


@pytest.mark.parametrize("name", sorted(SPECS))
def test_torch_expression_equals_the_float64_formula(name):
    spec = jit.ObjectiveSpec(*SPECS[name])
    g = torch.Generator().manual_seed(3)
    for D in (2, 5, 64):
        X = torch.rand(9, D, generator=g, dtype=torch.float64) * 10 - 5
        torch.testing.assert_close(spec.torch_fn(X), f64(name, X), rtol=1e-12, atol=1e-9)
    X32 = (torch.rand(4, 33, generator=g) * 4 - 2)
    out = spec.torch_fn(X32)
    assert out.dtype == torch.float32 and out.shape == (4,)


def test_integer_powers_expand_to_products_and_others_to_powf():
    src = jit.ObjectiveSpec({"s": "x**3 + x**-2 + x**0.5 + 2**x"}, "s").source
    assert "(x * x * x)" in src and "(1.0f / (x * x))" in src and "powf(x, 0.5f)" in src and "powf(2.0f, x)" in src
    body = [ln for ln in src.splitlines() if "s0 +=" in ln or "return" in ln]
    assert body and not any("__" in ln for ln in body)  # no fast-math intrinsics


# ------------------------------------------------------------------------------------------------ NVRTC
@pytest.fixture(scope="module")
def compiled():
    out = {}
    for name, (sums, value) in SPECS.items():
        t0 = time.perf_counter()
        out[name] = jit.compile_source(jit.ObjectiveSpec(sums, value).source)
        out[name].wall = time.perf_counter() - t0
    return out


@pytest.mark.parametrize("name", sorted(SPECS))
def test_nvrtc_compiles_every_kernel_for_sm90a_without_spills(compiled, name):
    c = compiled[name]
    assert c.cubin[:4] == b"\x7fELF" and len(c.names) == N_KERNELS == len(jit.kernel_expressions())
    assert set(c.kernel_info) == set(jit.kernel_expressions())
    for expr, info in c.kernel_info.items():
        assert info["spill_stores"] == 0 and info["spill_loads"] == 0, (name, expr, info)
        assert 0 < info["registers"] <= 255
    sample = [i["registers"] for e, i in c.kernel_info.items() if "sample_eval_kernel" in e]
    # the launch bounds (256 threads, 3 blocks per SM) leave at most 80 registers to the sampling kernels
    assert max(sample) <= 80
    print(f"{name}: sampling kernels {min(sample)}-{max(sample)} registers, compile {c.wall:.2f} s")


def test_generated_source_is_the_cache_key(lib):
    a = jit.compile_objective(jit.ObjectiveSpec({"s": "x*x + 0.125"}, "s"))
    b = jit.compile_objective(jit.ObjectiveSpec({"s": "x*x + 0.125"}, "s"))
    c = jit.compile_objective(jit.ObjectiveSpec({"s": "x*x + 0.25"}, "s"))
    assert a is b and c is not a and c.objective_id != a.objective_id


# ------------------------------------------------------------------------------------------------ the C ABI
def _names(n=N_KERNELS):
    return (ctypes.c_char_p * max(n, 1))(*[b"k"] * n)


def test_register_rejects_bad_arguments_without_a_device(lib):
    out = ctypes.c_int(-99)
    img = b"\x7fELF" + bytes(60)
    assert lib.evok_objective_register(None, len(img), _names(), N_KERNELS, ctypes.byref(out)) == E_NULLPTR
    assert lib.evok_objective_register(img, len(img), None, N_KERNELS, ctypes.byref(out)) == E_NULLPTR
    assert lib.evok_objective_register(img, len(img), _names(), N_KERNELS, None) == E_NULLPTR
    assert lib.evok_objective_register(img, 0, _names(), N_KERNELS, ctypes.byref(out)) == E_BADSIZE
    for n in (0, 1, N_KERNELS - 1, N_KERNELS + 1):
        assert lib.evok_objective_register(img, len(img), _names(n), n, ctypes.byref(out)) == E_BADSIZE
    holes = (ctypes.c_char_p * N_KERNELS)(*([b"k"] * (N_KERNELS - 1) + [None]))
    assert lib.evok_objective_register(img, len(img), holes, N_KERNELS, ctypes.byref(out)) == E_NULLPTR
    assert out.value == -99  # nothing registered


def test_ids_start_at_the_base_and_follow_registration_order(lib):
    img = b"\x7fELF" + bytes(60)  # registration stores the image; nothing loads it here
    ids = []
    for _ in range(3):
        out = ctypes.c_int(-1)
        assert lib.evok_objective_register(img, len(img), _names(), N_KERNELS, ctypes.byref(out)) == 0
        ids.append(out.value)
    assert ids[0] >= USER_BASE and ids == [ids[0], ids[0] + 1, ids[0] + 2]
    assert ids[2] < USER_BASE + USER_CAPACITY


def test_entry_points_refuse_unregistered_ids(lib):
    p = 64  # any non-null pointer: the argument checks never dereference it
    for oid in (-1, 4, 5, USER_BASE - 1, USER_BASE + USER_CAPACITY - 1, USER_BASE + USER_CAPACITY, 1 << 20):
        assert lib.evok_sample_eval(oid, p, 4, p, p, 0, 4, 4, 1, 0, 0, None, p, None) == E_BADENUM
        assert lib.evok_sample_eval_sq(oid, p, 4, p, p, 0, 4, 4, 0, 0, None, p, p, None) == E_BADENUM
        ptrs = (ctypes.c_void_p * 1)(p)
        assert lib.evok_sample_eval_push(oid, p, 4, p, p, 0, 4, 4, 1, 0, 0, None, 1, 0, ptrs, ptrs, p, p, None) == E_BADENUM
        assert lib.evok_eval(oid, p, 4, 4, 4, p, None) == E_BADENUM
        assert lib.evok_objective_load(oid) == E_BADENUM
    assert lib.evok_eval(0, p, 4, 4, 4, p, None) == E_BADENUM  # EVOK_OBJ_NONE evaluates nothing, as before
    assert b"lacks" in lib.evok_error_string(-7)


# ------------------------------------------------------------------------------------------------ the Python object
def test_fused_objective_is_a_vectorised_fitness_function_on_the_cpu(lib):
    from evotorch_b200 import Problem
    from evotorch_b200.objectives import FusedObjective

    st = FusedObjective("styblinski_tang", *SPECS["styblinski_tang"])
    assert st.__evotorch_vectorized__ and st.evok_objective_id >= USER_BASE and st.kernel_info
    X = torch.rand(6, 10, dtype=torch.float64) * 10 - 5
    torch.testing.assert_close(st(X), f64("styblinski_tang", X))
    torch.testing.assert_close(st(X[0]), f64("styblinski_tang", X[:1])[0])
    prob = Problem("min", st, solution_length=10, initial_bounds=(-5, 5), seed=0)
    batch = prob.generate_batch(8)
    prob.evaluate(batch)
    torch.testing.assert_close(batch.evals[:, 0].double(), f64("styblinski_tang", batch.values), rtol=1e-5, atol=1e-4)
    with pytest.raises(ValueError, match="built-in"):
        FusedObjective("sphere", {"s": "x**2"}, "s")


def test_fused_objective_pickles_as_its_expressions(lib):
    from evotorch_b200 import ops
    from evotorch_b200.objectives import FusedObjective

    a = FusedObjective("ackley2", *SPECS["ackley_twin"])
    b = pickle.loads(pickle.dumps(a))
    assert isinstance(b, FusedObjective) and b is not a
    assert (b.name, b.sums, b.value, b.evok_objective_id) == (a.name, a.sums, a.value, a.evok_objective_id)
    assert ops.OBJECTIVE_IDS["ackley2"] == a.evok_objective_id
    assert len(pickle.dumps(a)) < 1000  # the spec, not the cubin
