"""FusedObjective with pair terms (terms of x_j and its neighbour xn = x_{j+1}) without a GPU: the translator, the torch function
against hand-written float64 formulas, the generated source and the NVRTC compilation of every kernel for sm_90a."""

import math

import pytest
import torch

from evotorch_b200 import jit

N_KERNELS = 22

# the pair objectives of the tests (and of scripts/fused_objective_bench.py); the GPU tests use the same ones
PAIR_SPECS = {
    "rosenbrock": ({"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s"),
    "trid": ({"a": "(x - 1)**2", "b": "x * xn"}, "a - b"),
    "dixon_price": ({"a": "maximum(0, 1 - j) * (x - 1)**2", "b": "(j + 2) * (2*xn**2 - x)**2"}, "a + b"),
    "mix4": ({"p": "cos(xn - x)", "q": "(j/D) * (xn + x)**2", "r": "x**2", "t": "abs(x)"}, "r + q - p + sqrt(t)"),
}


def f64(name: str, X: torch.Tensor) -> torch.Tensor:
    """The objectives written out by hand in float64: a pair sum runs over j = 0 .. D-2."""
    X = X.double()
    D = X.shape[-1]
    x, xn = X[..., :-1], X[..., 1:]
    jp = torch.arange(D - 1, dtype=torch.float64, device=X.device)
    if name == "rosenbrock":
        return (100 * (xn - x**2) ** 2 + (1 - x) ** 2).sum(-1)
    if name == "trid":
        return ((X - 1) ** 2).sum(-1) - (x * xn).sum(-1)
    if name == "dixon_price":
        return (X[..., 0] - 1) ** 2 + ((jp + 2) * (2 * xn**2 - x) ** 2).sum(-1)
    return (X**2).sum(-1) + ((jp / D) * (xn + x) ** 2).sum(-1) - torch.cos(xn - x).sum(-1) + torch.sqrt(X.abs().sum(-1))


# ------------------------------------------------------------------------------------------------ the translator
@pytest.mark.parametrize("term", ["xn", "x * xn", "xn - x**2", "exp(-xn) + j * x / D", "minimum(xn, x)", "xn**0.5"])
def test_xn_is_accepted_in_terms(term):
    spec = jit.ObjectiveSpec({"s": term, "t": "x"}, "s + t")
    assert spec.pairs == {"s"}
    assert "kPairs = true" in spec.source and "add_pair(float x, float xn, int64_t j)" in spec.source


@pytest.mark.parametrize("value", ["s + xn", "xn", "sqrt(xn * s)"])
def test_xn_is_an_unknown_name_in_value(value):
    with pytest.raises(ValueError, match="unknown name 'xn'") as info:
        jit.ObjectiveSpec({"s": "x * xn"}, value)
    names = str(info.value).split("the names")[-1]
    assert "xn" not in names and "s" in names and "D" in names  # the message names what `value` may use


def test_the_term_message_names_xn():
    with pytest.raises(ValueError, match="unknown name 'y'") as info:
        jit.ObjectiveSpec({"s": "x * y"}, "s")
    assert "x, xn, j, D" in str(info.value)


def test_xn_may_name_a_sum():
    """Sum names live only in `value`, where xn is not a name: no clash, and a sum called xn stays accepted."""
    spec = jit.ObjectiveSpec({"xn": "x**2"}, "xn + 1")
    assert not spec.pairs and "add_pair" not in spec.source


@pytest.mark.parametrize("name", sorted(PAIR_SPECS))
def test_torch_function_equals_the_float64_formula(name):
    spec = jit.ObjectiveSpec(*PAIR_SPECS[name])
    g = torch.Generator().manual_seed(11)
    for D in (1, 2, 3, 5, 64):
        X = torch.rand(9, D, generator=g, dtype=torch.float64) * 6 - 3
        torch.testing.assert_close(spec.torch_fn(X), f64(name, X), rtol=1e-12, atol=1e-9)
    X32 = torch.rand(4, 33, generator=g) * 4 - 2
    out = spec.torch_fn(X32)
    assert out.dtype == torch.float32 and out.shape == (4,)


def test_a_pair_sum_is_empty_at_D_1():
    X = torch.tensor([[0.5], [-2.0]], dtype=torch.float64)
    assert torch.equal(jit.ObjectiveSpec({"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s + 7").torch_fn(X), torch.full((2,), 7.0, dtype=torch.float64))
    # the element sum of the same objective still runs over the single column
    torch.testing.assert_close(jit.ObjectiveSpec({"a": "x**2", "b": "x * xn"}, "a + b").torch_fn(X), X[:, 0] ** 2)


def test_pair_terms_see_j_of_x_and_batch_dimensions():
    spec = jit.ObjectiveSpec({"s": "j * xn"}, "s")
    X = torch.arange(1.0, 7.0, dtype=torch.float64).reshape(1, 2, 3).expand(4, 2, 3)
    want = torch.tensor([0 * 2 + 1 * 3, 0 * 5 + 1 * 6], dtype=torch.float64).expand(4, 2)
    assert torch.equal(spec.torch_fn(X), want)


def test_a_spec_without_xn_has_no_pair_code():
    for sums, value in (({"s": "x**2"}, "s"), ({"a": "x**2", "c": "cos(2*pi*x)"}, "10*D + a - 10*c"), ({"s": "j * x"}, "s")):
        src = jit.ObjectiveSpec(sums, value).source
        assert "kPairs" not in src and "add_pair" not in src and "xn" not in src


def test_pair_and_element_terms_go_to_their_own_functions():
    src = jit.ObjectiveSpec(*PAIR_SPECS["mix4"]).source
    add = src.split("void add(")[1].split("}")[0]
    pair = src.split("void add_pair(")[1].split("}")[0]
    assert "s2 +=" in add and "s3 +=" in add and "s0" not in add and "s1" not in add and "jf" not in add
    assert "s0 +=" in pair and "s1 +=" in pair and "s2" not in pair and "const float jf = (float)j;" in pair
    assert "S_p = evok::warp_sum(s0)" in src and "S_t = evok::warp_sum(s3)" in src


# ------------------------------------------------------------------------------------------------ NVRTC
@pytest.fixture(scope="module")
def compiled():
    return {name: jit.compile_source(jit.ObjectiveSpec(*spec).source) for name, spec in PAIR_SPECS.items()}


@pytest.mark.parametrize("name", sorted(PAIR_SPECS))
def test_nvrtc_compiles_every_pair_kernel_for_sm90a_without_spills(compiled, name):
    c = compiled[name]
    assert c.cubin[:4] == b"\x7fELF" and len(c.names) == N_KERNELS
    assert set(c.kernel_info) == set(jit.kernel_expressions())
    for expr, info in c.kernel_info.items():
        assert info["spill_stores"] == 0 and info["spill_loads"] == 0, (name, expr, info)
    sample = [i["registers"] for e, i in c.kernel_info.items() if "sample_eval_kernel" in e]
    evals = [i["registers"] for e, i in c.kernel_info.items() if "eval_kernel<" in e and "sample" not in e]
    # the sampling kernels keep the built-in launch bounds (256 threads, 3 blocks per SM): at most 80 registers
    assert max(sample) <= 80 and math.isfinite(c.seconds)
    print(f"{name}: sampling kernels {min(sample)}-{max(sample)} registers, eval {min(evals)}-{max(evals)}, compile {c.seconds:.2f} s")
