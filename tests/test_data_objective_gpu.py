"""FusedObjective with data on the GPU: every kernel of the table against the float64 torch twin on the stored rows, isolation of
the data reads, the batched samplers with shared and per-item data, whole searchers (lazy, stored, graph replay), instances and
the ABI errors."""

import ctypes
import gc
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, jit, ops
    from evotorch_b200 import _native as nat
    from evotorch_b200.algorithms import CEM, CMAES, PGPE
    from evotorch_b200.algorithms.functional import pgpe, pgpe_ask_and_evaluate, pgpe_tell
    from evotorch_b200.algorithms.functional.misc import get_functional_optimizer
    from evotorch_b200.objectives import FusedObjective

DEV = "cuda"
E_BADSIZE, E_BADENUM, E_NODATA = -2, -3, -8
LSQ = ({"s": "w * (x - t)**2"}, "s + lam * D")
SHIFTED_RASTRIGIN = ({"s": "(x - o)**2 - 10 * cos(2 * pi * (x - o))"}, "10 * D + s")
SHIFTED_ROSENBROCK = ({"s": "100*((xn - o_n) - (x - o)**2)**2 + (1 - (x - o))**2"}, "s")
SHIFTED_SPHERE = ({"s": "(x - o)**2"}, "s")
NAN = float("nan")


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed + sum(shape))).to(DEV)


def in_nan(t, lead=4, pad=4):
    """A view with the values of t (..., L) inside a NaN buffer: `lead` floats before the first item (4: 16-byte aligned, 1: a
    4-byte offset) and `pad` NaNs between the items (4 keeps the items of a row length that is a multiple of 4 aligned), so a read
    outside [0, L) of an item meets a NaN."""
    L = t.shape[-1]
    items = max(t.numel() // L, 1)
    buf = torch.full((lead + items * (L + pad) + 8,), NAN, device=DEV)
    view = buf[lead:lead + items * (L + pad)].view(items, L + pad)[:, :L]
    view.copy_(t.reshape(items, L))
    return view.view(t.shape) if t.ndim > 1 else view[0]


def params(D, offset=False, seed=0):
    g = torch.Generator().manual_seed(seed + D)
    mu = (torch.rand(D + 1, generator=g) * 4 - 2).to(DEV)
    sg = (torch.rand(D + 1, generator=g) + 0.5).to(DEV)
    return (mu[1:], sg[1:]) if offset else (mu[:D].clone(), sg[:D].clone())


def objectives(D, lead=4, batch=()):
    """The three documented objectives on data of row length D kept inside NaN buffers."""
    o, w, lam = rnd(*batch, D, seed=1), rnd(*batch, D, seed=2).abs() + 0.1, rnd(*batch, 1, seed=3).abs()  # a sum of positive terms
    return {"lsq": FusedObjective("lsq", *LSQ, data={"t": in_nan(o, lead), "w": in_nan(w, lead), "lam": in_nan(lam, lead)}),
            "shifted_rastrigin": FusedObjective("shifted_rastrigin", *SHIFTED_RASTRIGIN, data={"o": in_nan(o, lead)}),
            "shifted_rosenbrock": FusedObjective("shifted_rosenbrock", *SHIFTED_ROSENBROCK, data={"o": in_nan(o, lead)})}


def close(f, obj, X, what):
    """f against the float64 torch twin on the rows X: a relative error of a few rounding errors per add of a row's sums, on the
    scale of the absolute terms (the Rastrigin cosines cancel), and no NaN."""
    ref = obj._torch_fn(X.double())
    D = X.shape[-1]
    tol = (D / 32 + 40) * 2.0**-23
    scale = ref.abs() + (20.0 * D if "rastrigin" in obj.name else 0.0) + 1e-3
    if "rosenbrock" in obj.name:  # the rounding of zn - z^2 is on the scale of |zn| + z^2, however small the difference
        z = X.double() - obj.data["o"].double().unsqueeze(-2)
        scale = scale + 0.1 * ((z[..., 1:].abs() + z[..., :-1] ** 2) ** 2).sum(-1)
    err = ((f.double() - ref).abs() / scale).max().item()
    assert bool(torch.isfinite(f).all()) and err <= tol, (what, err, tol)


# ------------------------------------------------------------------------------------------------ every kernel
@pytest.mark.parametrize("lead", [4, 1])
@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("D", [2, 3, 5, 8, 127, 128, 129, 130, 256, 1000, 1028])
def test_every_kernel_against_the_float64_twin(D, symmetric, offset, lead):
    """Stored and lazy sampling, the SQ sampler, evaluation of X and of a misaligned view of X: the vectorised kernels when
    D % 4 == 0 and mu, sigma and the data are aligned (lead = 4), the scalar-column ones otherwise.  The samples are the built-in
    sampler's bit for bit, lazy fitnesses are the stored ones, and the data sits in NaN buffers."""
    n = 2 * 19
    mu, sg = params(D, offset)
    kw = dict(n_rows=n, symmetric=symmetric, seed=0xDA7A + D, stream_id=2, row0=6)
    kq = {k: v for k, v in kw.items() if k != "symmetric"}
    Xb = torch.empty(n, D, device=DEV)
    ops.sample_eval(ops.OBJ_SPHERE, Xb, mu, sg, f=torch.empty(n, device=DEV), **kw)
    for name, o in objectives(D, lead).items():
        oid = o.evok_objective_id
        assert oid >= 1024
        X, f, fl = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        before = ops.launch_count()
        ops.sample_eval(oid, X, mu, sg, f=f, **kw)
        ops.sample_eval(oid, None, mu, sg, f=fl, **kw)
        fe = o(X)  # evok_eval
        fe_view = o(torch.empty(n, D + 1, device=DEV)[:, 1:].copy_(X))  # its scalar-column kernel
        assert ops.launch_count() == before + 4
        torch.cuda.synchronize()
        assert same(X, Xb) and same(fl, f), name
        for label, got in (("sampler", f), ("eval", fe), ("eval of a view", fe_view)):
            close(got, o, X, (name, label))
        if not symmetric:
            Xq, fq, q, flq, ql = (torch.empty(n, D, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV),
                                  torch.empty(n, device=DEV), torch.empty(n, device=DEV))
            ops.sample_eval_sq(oid, Xq, mu, sg, q, f=fq, **kq)
            ops.sample_eval_sq(oid, None, mu, sg, ql, f=flq, **kq)
            torch.cuda.synchronize()
            assert same(Xq, X) and same(fq, f) and same(flq, f) and same(ql, q), name


@pytest.mark.parametrize("D", [2, 5, 128, 10_001])
def test_shifted_rosenbrock_pairs(D):
    o = rnd(D, seed=5)
    f = FusedObjective("shifted_rosenbrock", *SHIFTED_ROSENBROCK, data={"o": in_nan(o)})
    plain = FusedObjective("rosenbrock", {"s": "100*(xn - x**2)**2 + (1 - x)**2"}, "s")
    mu, sg = params(D)
    n = 64
    X, fx = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
    for symmetric in (True, False):
        ops.sample_eval(f.evok_objective_id, X, mu, sg, n_rows=n, symmetric=symmetric, seed=7, stream_id=0, f=fx)
        torch.cuda.synchronize()
        close(fx, f, X, symmetric)
        close(f(X), f, X, "eval")
    # the optimum is at o + 1, and the shifted function of X is the plain one of X - o
    assert float(f((o + 1).contiguous()[None])[0]) < 1e-5
    torch.testing.assert_close(f(X), plain((X - o).contiguous()), rtol=1e-4, atol=1e-3)


def test_push_variant_with_data():
    pw_path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_peer_exchange_world.py")
    spec = importlib.util.spec_from_file_location("_peer_exchange_world", pw_path)
    pw = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(pw)
    for D, symmetric, lazy in ((37, True, False), (40, True, True), (37, False, True), (40, False, False)):
        o = objectives(D)["lsq"]
        N = 600
        counts = pw.shard_rows(N, 2, 0, symmetric)[2]
        world = pw.SimWorld(counts, D)
        mu, sg = params(D)
        world.poison()
        for r, px in enumerate(world.px):
            with world.on(r):
                Xr = None if lazy else torch.empty(counts[r], D, device=DEV)
                ops.sample_eval_push(o.evok_objective_id, Xr, mu, sg, n_rows=counts[r], symmetric=symmetric, seed=11, stream_id=7,
                                     row0=world.row0[r], peer=px)
        world.producers_done()
        for r, px in enumerate(world.px):
            with world.on(r):
                px.wait_fitness()
        world.check(1, 0)
        X, f = torch.empty(N, D, device=DEV), torch.empty(N, device=DEV)
        ops.sample_eval(o.evok_objective_id, X, mu, sg, n_rows=N, symmetric=symmetric, seed=11, stream_id=7, f=f)
        torch.cuda.synchronize()
        for px in world.px:
            assert same(px.f_all, f)
        close(f, o, X, (D, symmetric, lazy))


# ------------------------------------------------------------------------------------------------ the batched samplers
@pytest.mark.parametrize("per_item", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("D", [8, 10])
def test_batched_kernels_with_shared_and_per_item_data(D, symmetric, per_item):
    """Stored and lazy, for D % 4 == 0 and not: item b is one plain launch on stream b with item b's data, bit for bit, and its
    fitnesses are the float64 twin's.  Per-item rows are separated by NaN padding (an item stride of D + 4, which keeps the
    items aligned: D = 8 runs the vectorised kernels, D = 10 the scalar-column ones)."""
    B, n = 7, 12
    mu, sg = rnd(B, D, seed=20), rnd(B, D, seed=21).abs() + 0.5
    for name, o in objectives(D, batch=(B,) if per_item else ()).items():
        o.compile_batched()
        X, f, fl = torch.empty(B, n, D, device=DEV), torch.empty(B, n, device=DEV), torch.empty(B, n, device=DEV)
        ops.sample_eval_batched(o.evok_objective_id, X, mu, sg, f, symmetric=symmetric, seed=5)
        ops.sample_eval_batched(o.evok_objective_id, None, mu, sg, fl, symmetric=symmetric, seed=5)
        torch.cuda.synchronize()
        assert same(fl, f), name
        close(f, o, X, name)
        for b in (0, 3, B - 1):
            one = o.with_data(**{k: (t[b] if per_item else t).clone() for k, t in o.data.items()})
            Xb, fb = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
            ops.sample_eval(one.evok_objective_id, Xb, mu[b], sg[b], n_rows=n, symmetric=symmetric, seed=5, stream_id=b, f=fb)
            torch.cuda.synchronize()
            assert same(Xb, X[b]) and same(fb, f[b]), (name, b)


def test_more_items_than_one_grid_with_per_item_data():
    B, n, D = 65_600, 2, 4
    targets = rnd(B, D, seed=30)
    o = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": targets})
    o.compile_batched()
    mu, sg = torch.zeros(D, device=DEV), torch.ones(D, device=DEV)
    X, f = torch.empty(B, n, D, device=DEV), torch.empty(B, n, device=DEV)
    before = ops.launch_count()
    ops.sample_eval_batched(o.evok_objective_id, X, mu, sg, f, symmetric=True, seed=1)
    torch.cuda.synchronize()
    assert ops.launch_count() == before + 2  # two item chunks, the second starting at item 65 535 of the data
    torch.testing.assert_close(f.double(), ((X.double() - targets.double()[:, None]) ** 2).sum(-1), rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------ whole searchers
def _problem(objective, D, lazy=False):
    return Problem("min", objective, initial_bounds=(-2, 2), solution_length=D, device=DEV, seed=3, lazy_population=lazy)


SEARCHERS = {
    "pgpe": lambda p: PGPE(p, popsize=200, center_learning_rate=0.3, stdev_learning_rate=0.1, stdev_init=1.0),
    "cem": lambda p: CEM(p, popsize=120, parenthood_ratio=0.5, stdev_init=1.0),
    "sepcma": lambda p: CMAES(p, stdev_init=1.0, popsize=150, separable=True, center_init=torch.linspace(-1.5, 1.5, p.solution_length, device=DEV)),
}


def _state(s):
    return [s.m, s.sigma.reshape(-1)] if isinstance(s, CMAES) else [s._distribution.mu, s._distribution.sigma]


@pytest.mark.parametrize("name", list(SEARCHERS))
@pytest.mark.parametrize("D", [130, 260])
def test_searchers_graph_replay_lazy_and_a_data_update(name, D):
    """6 generations on the least-squares objective, whose target is overwritten (data['t'].copy_) after the third: graph replay
    equals eager stepping bit for bit, stored and lazy; a lazy run draws and evaluates the stored run's first population bit for
    bit and, for separable CMA-ES (whose lazy update sums in the stored order), follows it throughout.  The update shows in the
    fitnesses of the next generation: they are the float64 twin's on the new target."""
    t0, t1, w, lam = rnd(D, seed=40), rnd(D, seed=41), rnd(D, seed=42).abs() + 0.1, torch.tensor([0.3], device=DEV)

    def run(lazy, graph):
        o = FusedObjective("lsq", *LSQ, data={"t": t0.clone(), "w": w, "lam": lam})
        s = SEARCHERS[name](_problem(o, D, lazy=lazy))
        if graph:
            s.enable_cuda_graph()
        hist = []
        for g in range(6):
            if g == 3:
                o.data["t"].copy_(t1)
            s.step()
            X, f = s.population.values.clone(), s.population.evals.clone()
            close(f[:, 0], o, X, (lazy, graph, g))
            hist.append([t.detach().clone() for t in _state(s)] + [f, X])
        torch.cuda.synchronize()
        if graph:
            assert s._graph is not None, "the generation was not captured"
        return hist

    runs = {(lazy, graph): run(lazy, graph) for lazy in (False, True) for graph in (False, True)}
    for lazy in (False, True):
        for g, (a, b) in enumerate(zip(runs[(lazy, False)], runs[(lazy, True)])):
            assert all(same(x, y) for x, y in zip(a, b)), (lazy, g)
    assert all(same(x, y) for x, y in zip(runs[(False, False)][0][-2:], runs[(True, False)][0][-2:]))
    if name == "sepcma":
        for g, (a, b) in enumerate(zip(runs[(False, False)], runs[(True, False)])):
            assert all(same(x, y) for x, y in zip(a, b)), g


def test_two_objectives_of_one_source_on_two_streams():
    D, n = 1024, 4096
    mu, sg = params(D)
    a = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": torch.full((D,), 1.0, device=DEV)})
    b = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": torch.full((D,), -2.0, device=DEV)})
    assert a.source == b.source and a.evok_objective_id != b.evok_objective_id
    X = torch.empty(n, D, device=DEV)
    ops.sample_eval(ops.OBJ_SPHERE, X, mu, sg, n_rows=n, symmetric=True, seed=3, stream_id=0, f=torch.empty(n, device=DEV))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    out = {0: [], 1: []}
    torch.cuda.synchronize()
    for rep in range(8):
        for k, o in enumerate((a, b)):
            with torch.cuda.stream(streams[k]):
                f = torch.empty(n, device=DEV)
                ops.sample_eval(o.evok_objective_id, None, mu, sg, n_rows=n, symmetric=True, seed=3, stream_id=0, f=f)
                out[k].append(f)
    torch.cuda.synchronize()
    for k, o in enumerate((a, b)):
        close(out[k][0], o, X, k)
        assert all(same(f, out[k][0]) for f in out[k])
    assert not same(out[0][0], out[1][0])


def test_instances_are_released():
    D = 8
    mu, sg = params(D)
    ids = set()
    f = torch.empty(4, device=DEV)
    for i in range(300):  # more than the 256 objectives that can be registered
        o = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": torch.full((D,), float(i), device=DEV)})
        ids.add(o.evok_objective_id)
        if i % 50 == 0:
            ops.sample_eval(o.evok_objective_id, None, mu, sg, n_rows=4, symmetric=True, seed=0, stream_id=0, f=f)
        released = o.evok_objective_id
        del o
        gc.collect()
        assert nat.lib().evok_objective_release(released) == E_BADENUM  # the finalizer has released it already
    torch.cuda.synchronize()
    assert len(ids) < 300  # released ids are reused


# ------------------------------------------------------------------------------------------------ end to end
def test_pgpe_finds_the_shift():
    D = 100
    target = rnd(D, seed=50) * 2
    o = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": target})
    p = Problem("min", o, initial_bounds=(0.0, 0.0), solution_length=D, device=DEV, seed=1)
    s = PGPE(p, popsize=400, center_learning_rate=0.4, stdev_learning_rate=0.1, stdev_init=1.0, center_init=torch.zeros(D, device=DEV))
    start = float((target**2).sum().sqrt())
    s.run(300)
    dist = float((s._distribution.mu - target).norm())
    print(f"distance to the shift: {start:.2f} -> {dist:.3f}")
    assert dist < 0.05 * start


def test_functional_batch_solves_one_target_per_item():
    B, D, n = 64, 20, 200
    targets = rnd(B, D, seed=60) * 2
    o = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": targets})
    for lazy in (False, True):
        st = pgpe(center_init=torch.zeros(D, device=DEV), center_learning_rate=0.3, stdev_learning_rate=0.1, objective_sense="min",
                  stdev_init=1.0)  # one unbatched state, broadcast to the 64 data sets by the first ask
        for g in range(250):
            values, evals = pgpe_ask_and_evaluate(st, popsize=n, objective=o, lazy=lazy)
            assert evals.shape == (B, n) and tuple(values.shape) == (B, n, D)
            st = pgpe_tell(st, values, evals)
        center = get_functional_optimizer(st.optimizer)[1](st.optimizer_state)
        d = torch.cdist(center, targets)  # [item, target]
        own = d.diagonal()
        others = d + torch.eye(B, device=DEV) * 1e9
        print(f"lazy={lazy}: worst distance to the own target {float(own.max()):.3f}, nearest other target {float(others.min()):.3f}")
        assert float(own.max()) < 1.0 and float(others.min()) > 3.0  # ClipUp keeps moving at its step size around the target


# ------------------------------------------------------------------------------------------------ ABI errors
def test_abi_errors_launch_nothing():
    D, n, B = 8, 4, 3
    lib = nat.lib()
    st = torch.cuda.current_stream().cuda_stream
    mu, sg = params(D)
    X, f = torch.empty(B, n, D, device=DEV), torch.full((B, n), -1.0, device=DEV)
    shared = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": rnd(D)})
    longer = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": rnd(D + 4)})
    per_item = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": rnd(B, D)})
    shared.compile_batched()
    base = jit.compile_objective(shared._spec).objective_id
    torch.cuda.synchronize()
    before = ops.launch_count()

    def plain(oid):
        return lib.evok_sample_eval(oid, X.data_ptr(), D, mu.data_ptr(), sg.data_ptr(), 0, n, D, 1, 0, 0, None, f.data_ptr(), st)

    def batched(oid, items):
        return lib.evok_sample_eval_batched(oid, X.data_ptr(), n * D, D, mu.data_ptr(), 0, sg.data_ptr(), 0, items, n, D, 1, 0, 0, f.data_ptr(), st)

    assert plain(longer.evok_objective_id) == E_BADSIZE  # a vector of another length than D
    assert lib.evok_eval(longer.evok_objective_id, X.data_ptr(), D, n, D, f.data_ptr(), st) == E_BADSIZE
    assert plain(per_item.evok_objective_id) == E_BADSIZE  # per-item data on an entry that is not batched
    assert lib.evok_eval(per_item.evok_objective_id, X.data_ptr(), D, n, D, f.data_ptr(), st) == E_BADSIZE
    assert batched(per_item.evok_objective_id, B - 1) == E_BADSIZE  # another number of items
    assert plain(base) == E_NODATA and batched(base, B) == E_NODATA  # the id that declares the data, without an instance
    assert lib.evok_eval(base, X.data_ptr(), D, n, D, f.data_ptr(), st) == E_NODATA
    assert plain(shared.evok_objective_id + 5000) == E_BADENUM  # no such instance
    with pytest.raises(ValueError, match="declares data"):
        ops.sample_eval(base, None, mu, sg, n_rows=n, symmetric=True, seed=0, stream_id=0, f=f[0])
    # instances: the declared count and kinds
    ptr, one, zero = (ctypes.c_void_p * 1)(X.data_ptr()), (ctypes.c_int64 * 1)(1), (ctypes.c_int64 * 1)(0)
    out = ctypes.c_int(-1)
    assert lib.evok_objective_instance(base, ptr, one, zero, 1, 1, ctypes.byref(out)) == E_BADSIZE  # a scalar for the declared vector
    assert lib.evok_objective_instance(ops.OBJ_SPHERE, ptr, one, zero, 1, 1, ctypes.byref(out)) == E_BADENUM
    no_data = FusedObjective("plain_sphere", {"s": "x**2"}, "s")
    assert lib.evok_objective_instance(no_data.evok_objective_id, ptr, one, zero, 1, 1, ctypes.byref(out)) == E_NODATA
    assert out.value == -1
    torch.cuda.synchronize()
    assert ops.launch_count() == before and bool((f == -1.0).all())
    # and the calls that are right
    # and the calls that are right (the batched image belongs to the source, so to every objective on it)
    assert batched(shared.evok_objective_id, B) == 0 and batched(per_item.evok_objective_id, B) == 0
    torch.cuda.synchronize()
    assert ops.launch_count() == before + 2


def test_data_on_another_device_is_refused():
    o = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": torch.zeros(8)})  # CPU data: no fused kernel
    assert o.evok_objective_id is None
    X = rnd(4, 8)
    torch.testing.assert_close(o(X), (X**2).sum(-1))
    if torch.cuda.device_count() > 1:
        far = FusedObjective("shifted_sphere", *SHIFTED_SPHERE, data={"o": torch.zeros(8, device="cuda:1")})
        with pytest.raises(ValueError, match="the data of the objective is on"):
            far(X)
