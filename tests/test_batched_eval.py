"""The batched evaluation without a device: return codes of evok_eval_batched and evok_objective_register_eval_batched (every
case returns before a device is touched, so nothing is launched), the order of its kernels, their NVRTC compile with no spills,
and the CPU fallbacks of evaluate_batched and cmaes_ask_and_evaluate."""

import ctypes

import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200 import jit
from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_ask_and_evaluate
from evotorch_b200.objectives import FusedObjective, rastrigin, sphere

NULLPTR, BADSIZE, BADENUM, NOKERNEL, NODATA = -1, -2, -3, -7, -8  # EVOK_E_* of include/evok.h
EVAL_BATCHED_KERNELS = 2
P = 64  # any non-null pointer: the argument checks never dereference it
IMG = b"\x7fELF" + bytes(60)


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def names(n, value=b"k"):
    return (ctypes.c_char_p * n)(*[value] * n)


def register(lib):
    out = ctypes.c_int(-1)
    assert lib.evok_objective_register(IMG, len(IMG), names(22), 22, ctypes.byref(out)) == 0
    return out.value


@pytest.fixture(scope="module")
def registered(lib):
    """Registered from a dummy image: [0] with a dummy batched evaluation image, [1] without, [2] with it and declared data
    (one vector), [3] an instance of [2] with per-item data for 3 items, [4] an instance of [2] with one data set."""
    ids = [register(lib) for _ in range(3)]
    for i in (0, 2):
        assert lib.evok_objective_register_eval_batched(ids[i], IMG, len(IMG), names(EVAL_BATCHED_KERNELS), EVAL_BATCHED_KERNELS) == 0
    assert lib.evok_objective_declare_data(ids[2], 1, (ctypes.c_int * 1)(1)) == 0
    for n_items in (3, 1):
        out = ctypes.c_int(-1)
        assert lib.evok_objective_instance(ids[2], (ctypes.c_void_p * 1)(P), (ctypes.c_int64 * 1)(8), (ctypes.c_int64 * 1)(8), n_items, 1,
                                           ctypes.byref(out)) == 0
        ids.append(out.value)
    return ids


BASE = dict(X=P, sx=16, ldx=8, items=2, n_rows=0, D=8, f=P)


def call(lib, objective, a):
    return lib.evok_eval_batched(objective, a["X"], a["sx"], a["ldx"], a["items"], a["n_rows"], a["D"], 0, 0, a["f"], None)


# (changed arguments, code for a built-in objective and a registered id with the batched evaluation image)
CASES = [
    ({}, 0),
    (dict(items=0, n_rows=5), 0),
    (dict(sx=0), 0),
    (dict(sx=3), 0),
    (dict(ldx=9), 0),
    (dict(X=None), NULLPTR),
    (dict(f=None), NULLPTR),
    (dict(f=None, D=0), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(n_rows=-1), BADSIZE),
    (dict(sx=-16), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(D=-4), BADSIZE),
    (dict(ldx=7), BADSIZE),
    (dict(ldx=7, items=0), BADSIZE),
]


@pytest.mark.parametrize("changes,code", CASES)
def test_eval_batched_codes(lib, registered, changes, code):
    a = dict(BASE, **changes)
    before = lib.evok_launch_count()
    for objective in (1, 2, 3, registered[0]):
        assert call(lib, objective, a) == code, objective
    # EVOK_OBJ_NONE, ids out of range and unregistered ids are refused after the null pointers
    for objective in (0, 4, 63, 64 + 255, -1, 1024 + 65535):
        assert call(lib, objective, a) == (NULLPTR if code == NULLPTR else BADENUM), objective
    # a registered id without the batched evaluation image: its kernels do not exist
    assert call(lib, registered[1], a) == (code if code != 0 else NOKERNEL)
    # a registered id that declares data is launched through an instance only
    assert call(lib, registered[2], a) == (code if code != 0 else NODATA)
    assert lib.evok_launch_count() == before


def test_eval_batched_data_codes(lib, registered):
    per_item, shared = registered[3], registered[4]
    before = lib.evok_launch_count()
    for n_items in (0, 1, 3):  # a binding of one data set serves any number of items
        assert call(lib, shared, dict(BASE, items=n_items)) == 0
    assert call(lib, per_item, dict(BASE, items=3)) == 0
    for n_items in (0, 1, 2, 4):  # per-item data for 3 items: a call on another number of items
        assert call(lib, per_item, dict(BASE, items=n_items)) == BADSIZE, n_items
    assert call(lib, per_item, dict(BASE, items=4, X=None)) == NULLPTR  # the null pointers come first
    assert call(lib, shared, dict(BASE, D=12, ldx=12)) == BADSIZE  # the vector has length 8
    assert lib.evok_launch_count() == before


def test_register_eval_batched_codes(lib, registered):
    ok = names(EVAL_BATCHED_KERNELS)
    reg = lib.evok_objective_register_eval_batched
    assert reg(registered[0], None, len(IMG), ok, EVAL_BATCHED_KERNELS) == NULLPTR
    assert reg(registered[0], IMG, len(IMG), None, EVAL_BATCHED_KERNELS) == NULLPTR
    with_null = (ctypes.c_char_p * EVAL_BATCHED_KERNELS)(b"k", None)
    assert reg(registered[0], IMG, len(IMG), with_null, EVAL_BATCHED_KERNELS) == NULLPTR
    assert reg(registered[0], IMG, 0, ok, EVAL_BATCHED_KERNELS) == BADSIZE
    for n in (0, 1, 3, 8, 22):
        assert reg(registered[0], IMG, len(IMG), names(n), n) == BADSIZE
    for objective in (0, 1, 2, 3, 4, 63, 64 + 255, -1, registered[3]):  # built-in ids, unregistered ids, an instance
        assert reg(objective, IMG, len(IMG), ok, EVAL_BATCHED_KERNELS) == BADENUM
    # the other images' counts are unchanged
    assert lib.evok_objective_register_batched(registered[0], IMG, len(IMG), ok, EVAL_BATCHED_KERNELS) == BADSIZE


def test_eval_batched_kernel_order():
    ex = jit.eval_batched_kernel_expressions()
    assert len(ex) == jit.N_EVAL_BATCHED_KERNELS == EVAL_BATCHED_KERNELS
    # EVOK_OBJ_KERNEL_EVAL_BATCHED + vec
    assert ex == ["evok::eval_batched_kernel<evok_user::Acc, false>", "evok::eval_batched_kernel<evok_user::Acc, true>"]
    assert jit.N_KERNELS == 22 and jit.N_BATCHED_KERNELS == 8


SPECS = {
    "element": dict(sums={"s": "x**4 - 16*x**2 + 5*x"}, value="0.5 * s"),
    "pair": dict(sums={"s": "100*(xn - x**2)**2 + (1 - x)**2"}, value="s"),
    "running": dict(running={"c": "x"}, sums={"s": "c**2"}, value="s"),
    "data": dict(sums={"s": "w * (x - t)**2"}, value="s + lam * D", kinds={"t": True, "w": True, "lam": False}),
    "noise": dict(sums={"s": "(x + 0.1 * randn())**2", "u": "rand() * abs(x)"}, value="s + u + randn() + rand()"),
}


@pytest.mark.parametrize("name", sorted(SPECS))
def test_nvrtc_compiles_the_eval_batched_kernels(name):
    kw = dict(SPECS[name])
    s = jit.ObjectiveSpec(kw.pop("sums"), kw.pop("value"), kw.pop("kinds", None), **kw)
    if name == "noise":
        assert s.noisy and s.element_draws.normal and s.value_draws.normal
    c = jit.compile_source(s.source, jit.eval_batched_kernel_expressions())
    assert len(c.names) == EVAL_BATCHED_KERNELS and len(c.kernel_info) == EVAL_BATCHED_KERNELS
    for e, info in c.kernel_info.items():
        assert info["spill_stores"] == 0 and info["spill_loads"] == 0, (e, info)


# ------------------------------------------------------------------------------------------------ CPU fallbacks
@pytest.mark.parametrize("batch", [(), (3,), (2, 2)])
def test_cmaes_fallback_equals_ask_then_objective(batch):
    center = torch.linspace(-2, 2, 6, dtype=torch.float64).expand(batch + (6,)).clone()
    state = cmaes(center_init=center, stdev_init=0.5, objective_sense="min", popsize=7)
    torch.manual_seed(11)
    values, evals = cmaes_ask_and_evaluate(state, objective=rastrigin)
    torch.manual_seed(11)
    ref = cmaes_ask(state)
    assert values.dtype == torch.float64 and torch.equal(values, ref)
    assert torch.equal(evals, rastrigin(ref)) and evals.shape == batch + (7,)


def test_cmaes_fallback_with_per_item_data():
    t = torch.randn(3, 5, dtype=torch.float32)
    obj = FusedObjective("shifted_sphere_cpu", sums={"s": "(x - t)**2"}, value="s", data={"t": t})
    state = cmaes(center_init=torch.zeros(3, 5, dtype=torch.float64), stdev_init=1.0, objective_sense="min", popsize=6)
    torch.manual_seed(2)
    values, evals = cmaes_ask_and_evaluate(state, objective=obj)
    torch.manual_seed(2)
    ref = cmaes_ask(state)
    assert torch.equal(values, ref)
    assert torch.equal(evals, obj(ref))
    assert torch.allclose(evals, ((ref - t.double()[:, None, :]) ** 2).sum(-1))


def test_data_batch_shape_must_match():
    t = torch.zeros(4, 3)
    obj = FusedObjective("shifted_sphere_cpu4", sums={"s": "(x - t)**2"}, value="s", data={"t": t})
    state = cmaes(center_init=torch.zeros(2, 3, dtype=torch.float64), stdev_init=1.0, objective_sense="min")
    with pytest.raises(ValueError, match=r"batch shape \(4,\).*\(2,\)"):
        cmaes_ask_and_evaluate(state, objective=obj)
    with pytest.raises(ValueError, match=r"batch shape \(4,\).*\(2,\)"):
        obj.evaluate_batched(torch.zeros(2, 5, 3))
    with pytest.raises(ValueError, match=r"\(\.\.\., n, D\)"):
        sphere.evaluate_batched(torch.zeros(3))


@pytest.mark.parametrize("objective", [sphere, rastrigin], ids=["sphere", "rastrigin"])
def test_evaluate_batched_cpu_is_the_torch_function(objective):
    x = torch.randn(2, 3, 5, 4, dtype=torch.float64)
    f = objective.evaluate_batched(x, seed=5)
    assert f.shape == (2, 3, 5) and torch.equal(f, objective(x))
