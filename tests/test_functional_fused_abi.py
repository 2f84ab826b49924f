"""The batched sample-and-evaluate entry points without a device: return codes of evok_sample_eval_batched,
evok_grad_batched_regen and evok_objective_register_batched (every case returns before a device is touched, so nothing is
launched), the Python fallbacks of pgpe_ask_and_evaluate / cem_ask_and_evaluate, and the NVRTC compile of the 8 batched
kernels."""

import ctypes

import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200 import jit
from evotorch_b200.algorithms.functional import cem, cem_ask, cem_ask_and_evaluate, pgpe, pgpe_ask, pgpe_ask_and_evaluate
from evotorch_b200.objectives import rastrigin

NULLPTR, BADSIZE, BADENUM, ODDROWS, NOKERNEL = -1, -2, -3, -5, -7  # EVOK_E_* of include/evok.h
BATCHED_KERNELS = 8
P = 64  # any non-null pointer: the argument checks never dereference it
ELEMENT_SPEC = ({"s": "x**4 - 16*x**2 + 5*x"}, "0.5 * s")
PAIR_SPEC = ({"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s")


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def names(n, value=b"k"):
    return (ctypes.c_char_p * n)(*[value] * n)


@pytest.fixture(scope="module")
def registered(lib):
    """Two ids registered from a dummy image: the first gets a dummy batched image too, the second none."""
    img = b"\x7fELF" + bytes(60)
    ids = []
    for _ in range(2):
        out = ctypes.c_int(-1)
        assert lib.evok_objective_register(img, len(img), names(22), 22, ctypes.byref(out)) == 0
        ids.append(out.value)
    assert lib.evok_objective_register_batched(ids[0], img, len(img), names(BATCHED_KERNELS), BATCHED_KERNELS) == 0
    return ids


SAMPLE_BASE = dict(X=P, sx=0, ldx=8, mu=P, sm=0, sigma=P, ss=0, items=2, n_rows=0, D=8, sym=1, f=P)


def sample_call(lib, objective, a):
    return lib.evok_sample_eval_batched(objective, a["X"], a["sx"], a["ldx"], a["mu"], a["sm"], a["sigma"], a["ss"], a["items"], a["n_rows"],
                                        a["D"], a["sym"], 0, 0, a["f"], None)


# (changed arguments, code for a built-in fused objective and the registered id with a batched image)
SAMPLE_CASES = [
    ({}, 0),
    (dict(X=None), 0),
    (dict(X=None, ldx=0), 0),
    (dict(X=None, sx=-8), 0),
    (dict(mu=None), NULLPTR),
    (dict(sigma=None), NULLPTR),
    (dict(f=None), NULLPTR),
    (dict(f=None, D=0), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(n_rows=-2), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(ldx=7), BADSIZE),
    (dict(sx=-8), BADSIZE),
    (dict(sm=-8), BADSIZE),
    (dict(ss=-8), BADSIZE),
    (dict(n_rows=3), ODDROWS),
    (dict(n_rows=3, sym=0, items=0), 0),
    (dict(n_rows=3, ldx=7), BADSIZE),
    (dict(items=0, n_rows=3), ODDROWS),
]


@pytest.mark.parametrize("changes,code", SAMPLE_CASES)
def test_sample_eval_batched_codes(lib, registered, changes, code):
    a = dict(SAMPLE_BASE, **changes)
    before = lib.evok_launch_count()
    for objective in (1, 2, 3, registered[0]):
        assert sample_call(lib, objective, a) == code, objective
    # EVOK_OBJ_NONE goes through evok_sample_batched; an id that names no objective is refused after the null pointers
    for objective in (0, 4, 63, 64 + 255):
        assert sample_call(lib, objective, a) == (NULLPTR if code == NULLPTR else BADENUM), objective
    # a registered id without a batched image: its kernels do not exist, and nothing is launched
    assert sample_call(lib, registered[1], a) == (code if code != 0 else NOKERNEL)
    assert lib.evok_launch_count() == before


GRAD_BASE = dict(form=1, w=P, mu=P, sm=0, sigma=P, ss=0, items=2, n_rows=4, D=8, out_mu=P, out_sigma=P, ws=P, ws_bytes=0)

GRAD_CASES = [
    (dict(items=0), 0),
    (dict(w=None), NULLPTR),
    (dict(mu=None), NULLPTR),
    (dict(sigma=None), NULLPTR),
    (dict(out_mu=None), NULLPTR),
    (dict(out_sigma=None), NULLPTR),
    (dict(ws=None), NULLPTR),
    (dict(form=4), BADENUM),
    (dict(form=-1), BADENUM),
    (dict(form=4, items=-1), BADENUM),
    (dict(items=-1), BADSIZE),
    (dict(n_rows=-2), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(sm=-4), BADSIZE),
    (dict(ss=-4), BADSIZE),
    (dict(n_rows=3), ODDROWS),
    (dict(n_rows=3, items=0), ODDROWS),
    (dict(n_rows=3, form=0, items=0), 0),
]


@pytest.mark.parametrize("changes,code", GRAD_CASES)
def test_grad_batched_regen_codes(lib, changes, code):
    a = dict(GRAD_BASE, **changes)
    before = lib.evok_launch_count()
    rc = lib.evok_grad_batched_regen(a["form"], a["w"], a["mu"], a["sm"], a["sigma"], a["ss"], a["items"], a["n_rows"], a["D"], 0, 0, 1.0, 1.0,
                                     a["out_mu"], a["out_sigma"], a["ws"], a["ws_bytes"], None)
    assert rc == code
    assert lib.evok_launch_count() == before


# evok_grad_batched takes the same checks, and X with its item stride and row pitch
GRAD_BATCHED_CASES = GRAD_CASES + [
    (dict(X=None), NULLPTR),
    (dict(X=None, ldx=7), NULLPTR),
    (dict(ldx=7), BADSIZE),
    (dict(sx=-32), BADSIZE),
    (dict(sx=-32, items=0), BADSIZE),
    (dict(ldx=7, n_rows=3), BADSIZE),
]


@pytest.mark.parametrize("changes,code", GRAD_BATCHED_CASES)
def test_grad_batched_codes(lib, changes, code):
    a = {**GRAD_BASE, "X": P, "sx": 32, "ldx": 8, **changes}
    before = lib.evok_launch_count()
    rc = lib.evok_grad_batched(a["form"], a["X"], a["sx"], a["ldx"], a["w"], a["mu"], a["sm"], a["sigma"], a["ss"], a["items"], a["n_rows"], a["D"],
                               1.0, 1.0, a["out_mu"], a["out_sigma"], a["ws"], a["ws_bytes"], None)
    assert rc == code
    assert lib.evok_launch_count() == before


def test_register_batched_codes(lib, registered):
    img = b"\x7fELF" + bytes(60)
    ok = names(BATCHED_KERNELS)
    reg = lib.evok_objective_register_batched
    assert reg(registered[0], None, len(img), ok, BATCHED_KERNELS) == NULLPTR
    assert reg(registered[0], img, len(img), None, BATCHED_KERNELS) == NULLPTR
    with_null = (ctypes.c_char_p * BATCHED_KERNELS)(*([b"k"] * (BATCHED_KERNELS - 1) + [None]))
    assert reg(registered[0], img, len(img), with_null, BATCHED_KERNELS) == NULLPTR
    assert reg(registered[0], img, 0, ok, BATCHED_KERNELS) == BADSIZE
    for n in (0, 7, 9, 22):
        assert reg(registered[0], img, len(img), names(n), n) == BADSIZE
    for objective in (0, 1, 2, 3, 4, 63, 64 + 255, -1):  # built-in ids and ids that name no registered objective
        assert reg(objective, img, len(img), ok, BATCHED_KERNELS) == BADENUM
    # the first image's count is unchanged: 22 kernels, and 8 is refused there
    out = ctypes.c_int(-1)
    assert lib.evok_objective_register(img, len(img), names(BATCHED_KERNELS), BATCHED_KERNELS, ctypes.byref(out)) == BADSIZE


def test_sample_eval_batched_python_checks(lib):
    from evotorch_b200 import ops

    with pytest.raises(ValueError, match="sample_batched"):
        ops.sample_eval_batched(ops.OBJ_NONE, None, torch.zeros(4), torch.ones(4), torch.zeros(2, 4), symmetric=False, seed=0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("batch", [(), (3,)])
def test_pgpe_fallback_equals_ask_then_objective(dtype, batch):
    center = torch.linspace(-2, 2, 8, dtype=dtype).expand(batch + (8,)).clone()
    state = pgpe(center_init=center, center_learning_rate=0.1, stdev_learning_rate=0.1, stdev_init=0.5, objective_sense="min")
    torch.manual_seed(7)
    values, evals = pgpe_ask_and_evaluate(state, popsize=6, objective=rastrigin)
    torch.manual_seed(7)
    ref = pgpe_ask(state, popsize=6)
    assert torch.equal(values, ref)
    assert torch.equal(evals, rastrigin(ref))
    assert evals.shape == batch + (6,)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cem_fallback_equals_ask_then_objective(dtype):
    state = cem(center_init=torch.zeros(2, 5, dtype=dtype), stdev_init=1.0, parenthood_ratio=0.5, objective_sense="max")
    f = lambda x: -(x**2).sum(-1)  # noqa: E731
    torch.manual_seed(3)
    values, evals = cem_ask_and_evaluate(state, popsize=7, objective=f)
    torch.manual_seed(3)
    ref = cem_ask(state, popsize=7)
    assert torch.equal(values, ref) and torch.equal(evals, f(ref))


def test_lazy_needs_the_fused_sampler():
    state = pgpe(center_init=torch.zeros(4), center_learning_rate=0.1, stdev_learning_rate=0.1, stdev_init=0.5, objective_sense="min")
    with pytest.raises(ValueError, match="no fused kernel"):
        pgpe_ask_and_evaluate(state, popsize=4, objective=lambda x: x.sum(-1), lazy=True)
    with pytest.raises(ValueError, match="float32 CUDA"):
        pgpe_ask_and_evaluate(state, popsize=4, objective=rastrigin, lazy=True)  # on the CPU
    cstate = cem(center_init=torch.zeros(4), stdev_init=1.0, parenthood_ratio=0.5, objective_sense="min")
    with pytest.raises(ValueError, match="lazy=True"):
        cem_ask_and_evaluate(cstate, popsize=4, objective=lambda x: x.sum(-1), lazy=True)


def test_batched_kernel_order():
    ex = jit.batched_kernel_expressions()
    assert len(ex) == jit.N_BATCHED_KERNELS == BATCHED_KERNELS
    # EVOK_OBJ_KERNEL_BATCHED + 4 sym + 2 store + vec
    for i, e in enumerate(ex):
        sym, store, vec = bool(i & 4), bool(i & 2), bool(i & 1)
        assert e == f"evok::sample_eval_batched_kernel<evok_user::Acc, {str(sym).lower()}, {str(store).lower()}, {str(vec).lower()}>"
    assert len(jit.kernel_expressions()) == jit.N_KERNELS == 22


@pytest.mark.parametrize("spec", [ELEMENT_SPEC, PAIR_SPEC], ids=["element", "pair"])
def test_nvrtc_compiles_the_batched_kernels(spec):
    s = jit.ObjectiveSpec(*spec)
    c = jit.compile_source(s.source, jit.batched_kernel_expressions())
    assert len(c.names) == BATCHED_KERNELS and len(c.kernel_info) == BATCHED_KERNELS
    for e, info in c.kernel_info.items():
        assert info["registers"] <= 80, (e, info)
        assert info["spill_stores"] == 0 and info["spill_loads"] == 0, (e, info)
