"""The batched evaluation on the GPU: every item of evok_eval_batched bit for bit against evok_eval_keyed on that item's rows (with
stream id stream_id0 + b, on the same path), across objectives, row lengths, layouts, item counts past the grid limit and NaN
canaries; populations stored by the batched sampler evaluated again to the sampler's fitnesses; and cmaes_ask_and_evaluate
against cmaes_ask and per-item keyed evaluation."""

import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import ops
    from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_ask_and_evaluate, cmaes_tell
    from evotorch_b200.algorithms.functional.misc import draw_philox_seed
    from evotorch_b200.objectives import FusedObjective, ackley, rastrigin, sphere

DEV = "cuda"
SEED, SID0 = 0x0BAD_5EED_0000_1234, 7
DIMS = [1, 3, 4, 31, 128, 129, 1000, 4097]


def _load(filename):
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), filename)
    spec = importlib.util.spec_from_file_location("_" + filename[:-3], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


NOISY = _load("test_noisy_objective.py")

SPECS = {
    "pair": dict(sums={"s": "100*(xn - x**2)**2 + (1 - x)**2"}, value="s"),
    "prod_max_min": dict(sums={"s": "x**2"}, prods={"p": "cos(x / sqrt(j + 1))"}, maxs={"m": "abs(x)"}, mins={"n": "x"},
                         value="1 + s / 4000 - p + m - n"),
    "running": dict(running={"c": "x"}, sums={"s": "c**2"}, value="s"),
    "where": dict(sums={"s": "where(x < 0, x**2, abs(x))"}, value="s"),
    "noise": dict(sums={"s": "(x + 0.1 * randn())**2", "u": "rand() * abs(x)"}, value="s + u + randn() + rand()"),
}
DATA_SPEC = dict(sums={"s": "(x - t)**2 + lam * x"}, value="s + lam")
_objs = {}


def same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def obj(name):
    if name not in _objs:
        _objs[name] = {"sphere": lambda: sphere, "rastrigin": lambda: rastrigin, "ackley": lambda: ackley}.get(
            name, lambda: FusedObjective("bev_" + name, **SPECS[name]))()
    return _objs[name]


def data_obj(kind, B, D, twins=True):
    """(objective, per-item twins) of an objective with a vector and a scalar: shared by all items, or one set per item (twins:
    False for none, past the number of live instances)."""
    g = torch.Generator().manual_seed(B * 1000 + D)
    if kind == "shared":
        t, lam = torch.randn(D, generator=g).to(DEV), torch.rand(1, generator=g).to(DEV)
        o = FusedObjective("bev_data", data={"t": t, "lam": lam}, **DATA_SPEC)
        return o, [o] * B
    t, lam = torch.randn(B, D, generator=g).to(DEV), torch.rand(B, 1, generator=g).to(DEV)
    o = FusedObjective("bev_data", data={"t": t, "lam": lam}, **DATA_SPEC)
    return o, [o.with_data(t=t[b], lam=lam[b]) for b in range(B)] if twins else None


def layout(B, n, D, *, offset=0, sx=None, ldx=None, seed=0):
    """X (B, n, D) as a strided view of a NaN-filled buffer: the padding between rows and items is NaN, so a read outside the
    rows makes a fitness NaN."""
    ldx = D if ldx is None else ldx
    sx = n * ldx if sx is None else sx
    size = offset + max(B - 1, 0) * sx + max(n - 1, 0) * ldx + D + 8
    buf = torch.full((size,), float("nan"), device=DEV)
    X = buf.as_strided((B, n, D), (sx, ldx, 1), offset)
    g = torch.Generator(device=DEV).manual_seed(seed + D)
    if B and n:
        vals = torch.randn(B, n, D, device=DEV, generator=g) * 2
        if sx == 0:  # every item reads the same rows
            X[0].copy_(vals[0])
        else:
            X.copy_(vals)
    return X


def vec_path(X):
    B, n, D = X.shape
    sx, ldx = (X.stride(0) if B > 1 else 0), (X.stride(1) if n > 1 else D)
    return D % 4 == 0 and X.data_ptr() % 16 == 0 and ldx % 4 == 0 and sx % 4 == 0


def single(oid, rows, vec, sid):
    """evok_eval_keyed on a copy of `rows` (n, D) on the given path: aligned for the vectorised one, at a one-float offset (an
    unaligned base) for the scalar one."""
    n, D = rows.shape
    if vec:
        Xs = rows.contiguous().clone()
    else:
        Xs = torch.empty(n * D + 1, device=DEV)[1:].view(n, D)
        Xs.copy_(rows)
    return ops.evaluate_keyed(oid, Xs, seed=SEED, stream_id=sid)


def batched(o, X):
    """evaluate_batched into an f with a NaN canary after the last item; checks the canary."""
    B, n, _ = X.shape
    if hasattr(o, "compile_eval_batched"):
        o.compile_eval_batched()
    fbuf = torch.full((B * n + 32,), float("nan"), device=DEV)
    f = ops.evaluate_batched(o.evok_objective_id, X, seed=SEED, stream_id0=SID0, f=fbuf[:B * n].view(B, n))
    torch.cuda.synchronize()
    assert torch.isnan(fbuf[B * n:]).all()
    return f


def check_items(o, twins, X, items=None):
    f = batched(o, X)
    vec = vec_path(X)
    assert torch.isfinite(f).all()
    for b in range(X.shape[0]) if items is None else items:
        assert same(f[b], single(twins[b].evok_objective_id, X[b], vec, SID0 + b)), b


OBJECTIVES = ["sphere", "rastrigin", "ackley"] + sorted(SPECS)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("name", OBJECTIVES)
def test_items_are_keyed_single_evaluations(name, D):
    o = obj(name)
    X = layout(5, 7, D)
    check_items(o, [o] * 5, X)
    if D % 4 == 0:
        assert vec_path(X)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", ["shared", "per_item"])
def test_items_with_data(kind, D):
    o, twins = data_obj(kind, 5, D)
    check_items(o, twins, layout(5, 7, D))


# X one float past an aligned base; an item stride that is not a multiple of 4 (aligned rows otherwise); every item on the
# same rows; a row pitch with NaN padding after every row
LAYOUTS = {
    "offset": lambda D: dict(offset=1),
    "item_stride_odd": lambda D: dict(ldx=D + 4 - D % 4, sx=7 * (D + 4 - D % 4) + 2),
    "item_stride_0": lambda D: dict(sx=0),
    "row_pitch": lambda D: dict(ldx=D + 8),
}


@pytest.mark.parametrize("where", sorted(LAYOUTS))
@pytest.mark.parametrize("D", [4, 129, 1000])
@pytest.mark.parametrize("name", ["rastrigin", "pair", "noise", "per_item"])
def test_layouts(name, D, where):
    X = layout(5, 7, D, **LAYOUTS[where](D))
    if name == "per_item":
        o, twins = data_obj("per_item", 5, D)
    else:
        o = obj(name)
        twins = [o] * 5
    check_items(o, twins, X)
    if where in ("offset", "item_stride_odd"):
        assert not vec_path(X)


@pytest.mark.parametrize("n", [0, 1])
@pytest.mark.parametrize("name", ["sphere", "noise"])
def test_zero_and_one_rows(name, n):
    o = obj(name)
    X = layout(5, n, 128)
    f = batched(o, X)
    assert f.shape == (5, n)
    for b in range(5):
        if n:
            assert same(f[b], single(o.evok_objective_id, X[b], True, SID0 + b))


@pytest.mark.parametrize("B", [1, 5])
def test_item_counts(B):
    o, twins = data_obj("per_item", B, 36)
    check_items(o, twins, layout(B, 9, 36))


@pytest.mark.parametrize("name", ["rastrigin", "noise"])
def test_items_across_the_chunk(name):
    """70 000 items: two launches of the 65535-item grid, the second on its own stream words and rows."""
    B, n, D = 70_000, 3, 8
    o = obj(name)
    X = layout(B, n, D)
    f = batched(o, X)
    assert torch.isfinite(f).all()
    if not getattr(o, "noisy", False):  # no key: one launch over all rows is every item's evaluation
        assert same(f.view(-1), ops.evaluate(o.evok_objective_id, X.reshape(B * n, D)))
    for b in (0, 1, 65_534, 65_535, 65_536, B - 1):
        assert same(f[b], single(o.evok_objective_id, X[b], True, SID0 + b)), b


def test_items_across_the_chunk_with_per_item_data():
    B, n, D = 66_000, 2, 4
    o, _ = data_obj("per_item", B, D, twins=False)
    X = layout(B, n, D)
    f = batched(o, X)
    for b in (0, 65_534, 65_535, B - 1):
        twin = o.with_data(t=o.data["t"][b], lam=o.data["lam"][b])
        assert same(f[b], single(twin.evok_objective_id, X[b], True, SID0 + b)), b


# ------------------------------------------------------------------------------------------------ stored populations
@pytest.mark.parametrize("symmetric", [False, True])
@pytest.mark.parametrize("name", ["input_noise_sphere", "where_noise", "running_pair_noise", "f7", "rastrigin"])
def test_stored_populations_get_their_fitnesses_again(name, symmetric):
    if name != "rastrigin" and "noisy_" + name not in _objs:
        _objs["noisy_" + name] = NOISY.make(name)
    o = rastrigin if name == "rastrigin" else _objs["noisy_" + name]
    if hasattr(o, "compile_batched"):
        o.compile_batched()
    B, n, D = 4, 64, 260
    g = torch.Generator(device=DEV).manual_seed(5)
    mu, sg = torch.randn(B, D, device=DEV, generator=g), torch.rand(B, D, device=DEV, generator=g) + 0.5
    X, f = torch.empty(B, n, D, device=DEV), torch.empty(B, n, device=DEV)
    ops.sample_eval_batched(o.evok_objective_id, X, mu, sg, f, symmetric=symmetric, seed=SEED, stream_id0=SID0)
    if hasattr(o, "compile_eval_batched"):
        o.compile_eval_batched()
    fe = ops.evaluate_batched(o.evok_objective_id, X, seed=SEED, stream_id0=SID0)
    assert same(fe, f)


# ------------------------------------------------------------------------------------------------ CMA-ES
def test_cmaes_values_are_the_ask():
    state = cmaes(center_init=torch.randn(8, 16, device=DEV), stdev_init=0.7, objective_sense="min")
    torch.manual_seed(3)
    values, evals = cmaes_ask_and_evaluate(state, objective=rastrigin)
    torch.manual_seed(3)
    ref = cmaes_ask(state)
    assert torch.equal(values, ref)
    assert evals.shape == (8, state.popsize) and same(evals, rastrigin.evaluate_batched(ref, seed=0))


def _equal_states(a, b):
    for k in ("center", "sigma", "C", "A", "p_sigma", "p_c"):
        assert same(getattr(a, k), getattr(b, k)), k
    assert a.generation == b.generation


def test_cmaes_generations_equal_ask_then_keyed_evaluation():
    B, D = 6, 12
    g = torch.Generator().manual_seed(9)
    o_shift = torch.randn(B, D, generator=g).to(DEV)
    o = FusedObjective("bev_noisy_shift", sums={"s": "(x - o + 0.01 * randn())**2"}, value="s + 0.001 * randn()", data={"o": o_shift})
    twins = [o.with_data(o=o_shift[b]) for b in range(B)]
    s1 = s2 = cmaes(center_init=torch.zeros(B, D, device=DEV), stdev_init=1.0, objective_sense="min")
    torch.manual_seed(21)
    for _ in range(20):
        rng = torch.get_rng_state()
        values, evals = cmaes_ask_and_evaluate(s1, objective=o)
        s1 = cmaes_tell(s1, values, evals)
        torch.set_rng_state(rng)
        seed = draw_philox_seed()
        torch.set_rng_state(rng)
        ref = cmaes_ask(s2)
        assert torch.equal(values, ref)
        ref_evals = torch.stack([ops.evaluate_keyed(twins[b].evok_objective_id, ref[b], seed=seed, stream_id=b) for b in range(B)])
        assert same(evals, ref_evals)
        s2 = cmaes_tell(s2, ref, ref_evals)
        _equal_states(s1, s2)


def test_cmaes_per_item_shifted_sphere_moves_every_centre_to_its_shift():
    B, n, D = 64, 24, 32
    g = torch.Generator().manual_seed(4)
    shift = (torch.randn(B, D, generator=g) * 2).to(DEV)
    o = FusedObjective("bev_shifted_sphere", sums={"s": "(x - o)**2"}, value="s", data={"o": shift})
    state = cmaes(center_init=torch.zeros(B, D, device=DEV), stdev_init=1.0, objective_sense="min", popsize=n)
    d0 = (state.center - shift).norm(dim=-1)
    torch.manual_seed(0)
    for _ in range(100):
        values, evals = cmaes_ask_and_evaluate(state, objective=o)
        state = cmaes_tell(state, values, evals)
    d = (state.center - shift).norm(dim=-1)
    assert (d < 0.5 * d0).all(), (d / d0).max().item()


def test_cmaes_noise_is_reproducible_and_fresh_every_generation():
    o = FusedObjective("bev_pure_noise", sums={"s": "x"}, value="0 * s + randn()")
    state = cmaes(center_init=torch.zeros(4, 8, device=DEV), stdev_init=1.0, objective_sense="min")
    torch.manual_seed(17)
    _, e1 = cmaes_ask_and_evaluate(state, objective=o)
    _, e2 = cmaes_ask_and_evaluate(state, objective=o)
    torch.manual_seed(17)
    _, e1b = cmaes_ask_and_evaluate(state, objective=o)
    assert same(e1, e1b)
    assert not torch.equal(e1, e2)
    assert e1.std().item() > 0.5 and len(set(e1.view(-1).tolist())) == e1.numel()
