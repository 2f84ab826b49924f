"""FusedObjective on the GPU: the run-time compiled kernels against the built-in ones (bit for bit) and against the float64 torch
expression (per element, within an error bound), through every fused path of the package."""

import importlib.util
import itertools
import math
import os
import pickle

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, jit, ops
    from evotorch_b200 import _native as nat
    from evotorch_b200.algorithms import CEM, CMAES, PGPE, SNES
    from evotorch_b200.objectives import FusedObjective, sphere

DEV = "cuda"
DIMS = [1, 3, 4, 5, 127, 1000, 10_001]
E_NOKERNEL = -7
U = 2.0**-24
C_BOUND = 1.0  # the constant of the error bound, calibrated once: the worst measured error was 0.40 of it (H100)

SPECS = {
    "styblinski_tang": ({"s": "x**4 - 16*x**2 + 5*x"}, "0.5 * s"),
    "ellipsoid": ({"s": "1e6 ** (j / (D - 1)) * x**2"}, "s"),
    "rastrigin_twin": ({"a": "x**2", "c": "cos(2*pi*x)"}, "10*D + a - 10*c"),
    "ackley_twin": ({"a": "x**2", "c": "cos(2*pi*x)"}, "-20*exp(-0.2*sqrt(a/D)) - exp(c/D) + 20 + e"),
    "schwefel": ({"s": "x * sin(sqrt(abs(x)))"}, "418.9829 * D - s"),
}


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


_objs = {}


def obj(name):
    if name not in _objs:
        _objs[name] = FusedObjective("sphere_twin", {"s": "x**2"}, "s") if name == "sphere_twin" else FusedObjective(name, *SPECS[name])
    return _objs[name]


def params(D, offset=False, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + D)
    mu = ((torch.rand(D + 1, generator=g) * 4 - 2) * scale).to(DEV)
    sg = (torch.rand(D + 1, generator=g) + 0.5).to(DEV)
    # offset: one float into the allocation, so the vectorised path is not taken even when D % 4 == 0
    return (mu[1:], sg[1:]) if offset else (mu[:D].clone(), sg[:D].clone())


# ------------------------------------------------------------------------------------------------ samples and the sphere twin
@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("D", DIMS)
def test_samples_and_sphere_twin_are_bit_identical_to_the_builtin(D, symmetric, offset):
    """Every instantiation: materialised and lazy, symmetric and not, the SQ sampler (with q) and the stand-alone evaluation."""
    twin = obj("sphere_twin").evok_objective_id
    n = 2 * 37
    mu, sg = params(D, offset)
    kw = dict(n_rows=n, seed=0xABCDEF12345 + D, stream_id=5, row0=4)
    runs = {}
    for oid in (ops.OBJ_SPHERE, twin):
        X, f, fl = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        ops.sample_eval(oid, X, mu, sg, symmetric=symmetric, f=f, **kw)
        ops.sample_eval(oid, None, mu, sg, symmetric=symmetric, f=fl, **kw)
        r = dict(X=X, f=f, fl=fl, fe=ops.evaluate(oid, X), fe_odd=ops.evaluate(oid, torch.empty(n, D + 1, device=DEV)[:, 1:].copy_(X)))
        if not symmetric:
            Xq, fq, q, flq, ql = (torch.empty(n, D, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV),
                                  torch.empty(n, device=DEV), torch.empty(n, device=DEV))
            ops.sample_eval_sq(oid, Xq, mu, sg, q, f=fq, **kw)
            ops.sample_eval_sq(oid, None, mu, sg, ql, f=flq, **kw)
            r.update(Xq=Xq, fq=fq, q=q, flq=flq, ql=ql)
        runs[oid] = r
    torch.cuda.synchronize()
    a, b = runs[ops.OBJ_SPHERE], runs[twin]
    for k in a:
        assert same(a[k], b[k]), k
    if not symmetric:
        assert same(b["Xq"], b["X"]) and same(b["fq"], b["f"])


# ------------------------------------------------------------------------------------------------ whole searchers
def _problem(objective, D, lazy=False, seed=3):
    return Problem("min", objective, initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=seed, lazy_population=lazy)


SEARCHERS = {
    "pgpe": lambda p: PGPE(p, popsize=200, center_learning_rate=0.3, stdev_learning_rate=0.1, stdev_init=1.0),
    "pgpe_graph": lambda p: PGPE(p, popsize=200, center_learning_rate=0.3, stdev_learning_rate=0.1, stdev_init=1.0),
    "snes": lambda p: SNES(p, popsize=120, stdev_init=1.0),
    "cem": lambda p: CEM(p, popsize=120, parenthood_ratio=0.5, stdev_init=1.0),
    "sepcma": lambda p: CMAES(p, stdev_init=1.0, popsize=150, separable=True),
    "sepcma_graph": lambda p: CMAES(p, stdev_init=1.0, popsize=150, separable=True),
    "cmaes": lambda p: CMAES(p, stdev_init=1.0, popsize=64),
}
CASES = [("pgpe", False), ("pgpe", True), ("pgpe_graph", False), ("snes", False), ("cem", False), ("sepcma", False), ("sepcma", True),
         ("sepcma_graph", False), ("sepcma_graph", True), ("cmaes", False)]


def _state(s):
    if isinstance(s, CMAES):
        return [s.m, s.sigma.reshape(-1)] + ([s.C] if hasattr(s, "C") else [])
    d = s._distribution
    return [d.mu, d.sigma]


@pytest.mark.parametrize("name,lazy", CASES)
def test_searcher_trajectories_equal_the_builtin_sphere(name, lazy):
    D = 37 if name == "cmaes" else 130
    runs = []
    for objective in (sphere, obj("sphere_twin")):
        s = SEARCHERS[name](_problem(objective, D, lazy=lazy))
        if name.endswith("_graph"):
            s.enable_cuda_graph()
        hist = []
        for _ in range(6):
            s.step()
            hist.append([t.detach().clone() for t in _state(s)] + [s.population.evals.clone()])
        runs.append(hist)
    torch.cuda.synchronize()
    for g, (a, b) in enumerate(zip(*runs)):
        for x, y in zip(a, b):
            assert same(x, y), f"generation {g}"


# ------------------------------------------------------------------------------------------------ error bound
def _err(node, env, names):
    """(value, error bound in units of 2^-24) of a parsed expression, in float64, first order."""
    import ast

    if isinstance(node, ast.Expression):
        return _err(node.body, env, names)
    if isinstance(node, ast.Constant):
        v = torch.as_tensor(float(node.value), dtype=torch.float64, device=DEV)
        return v, v.abs()
    if isinstance(node, ast.Name):
        if node.id in ("pi", "e"):
            v = torch.as_tensor(getattr(math, node.id), dtype=torch.float64, device=DEV)
            return v, v.abs()
        return env[node.id]
    if isinstance(node, ast.UnaryOp):
        v, e = _err(node.operand, env, names)
        return -v, e
    if isinstance(node, ast.BinOp):
        a, ea = _err(node.left, env, names)
        if isinstance(node.op, ast.Pow):
            n = jit._int_exponent(node.right)
            if n is not None and n > 0:
                v = a**n
                return v, n * (a.abs() ** (n - 1)) * ea + (n - 1) * v.abs()
            b, eb = _err(node.right, env, names)
            v = a**b
            return v, (b * a ** (b - 1)).abs() * ea + (torch.log(a.abs()) * v).abs() * eb + 3 * v.abs()
        b, eb = _err(node.right, env, names)
        if isinstance(node.op, ast.Add):
            v = a + b
            return v, ea + eb + v.abs()
        if isinstance(node.op, ast.Sub):
            v = a - b
            return v, ea + eb + v.abs()
        if isinstance(node.op, ast.Mult):
            v = a * b
            return v, ea * b.abs() + eb * a.abs() + v.abs()
        v = a / b
        return v, ea / b.abs() + eb * (a / (b * b)).abs() + v.abs()
    if isinstance(node, ast.Call):
        a, ea = _err(node.args[0], env, names)
        fn = node.func.id
        f, d = {"sqrt": (torch.sqrt, lambda a: 0.5 / torch.sqrt(a)), "exp": (torch.exp, torch.exp), "log": (torch.log, lambda a: 1 / a),
                "sin": (torch.sin, torch.cos), "cos": (torch.cos, torch.sin), "abs": (torch.abs, lambda a: torch.ones_like(a))}[fn]
        v = f(a)
        return v, d(a).abs() * ea + 2 * v.abs()
    raise AssertionError(node)


def reference_and_bound(name, X, D_value=None, drop=None, shift_j=0):
    """float64 f and its error bound for the rows X (float32 values), with optional mutations of the reference."""
    import ast

    sums, value = SPECS[name]
    X = X.double()
    n, D = X.shape
    Dv = float(D if D_value is None else D_value)
    zero = torch.zeros_like(X)
    env = {"x": (X, zero), "j": ((torch.arange(D, dtype=torch.float64, device=DEV) + shift_j).expand_as(X), zero),
           "D": (torch.full_like(X, float(D)), zero)}
    k_eff = math.ceil(D / 32) + 5  # per-lane sums, then five shuffle rounds
    S, eS = {}, {}
    for s, t in sums.items():
        v, e = _err(ast.parse(t, mode="eval"), env, None)
        v, e = torch.broadcast_to(v, X.shape), torch.broadcast_to(e, X.shape)
        S[s] = v.sum(1) * (0 if drop == s else 1)
        eS[s] = e.sum(1) + k_eff * v.abs().sum(1)
    tree = ast.parse(value, mode="eval")
    base = {s: (S[s], torch.zeros_like(S[s])) for s in S}
    base["D"] = (torch.full((n,), Dv, dtype=torch.float64, device=DEV), torch.zeros(n, dtype=torch.float64, device=DEV))
    f, e_value = _err(tree, base, None)
    # the sums' errors carried through `value` at the corners of their intervals
    carried = torch.zeros_like(f)
    for signs in itertools.product((-1.0, 1.0), repeat=len(S)):
        corner = {s: (S[s] + sg * C_BOUND * U * eS[s], torch.zeros_like(S[s])) for s, sg in zip(S, signs)}
        corner["D"] = base["D"]
        carried = torch.maximum(carried, (_err(tree, corner, None)[0] - f).abs())
    return f, C_BOUND * U * e_value + carried  # the corner deviation is already an absolute error


def _check_bound(name, X, f, **mut):
    ref, bound = reference_and_bound(name, X, **mut)
    err = (f.double() - ref).abs()
    return bool((err <= bound).all()), float((err / bound.clamp_min(1e-300)).max())


CASES_OBJ = [(name, D, sym, lazy) for name in SPECS for D in (3, 64, 1000, 10_001) for sym in (True, False) for lazy in (False, True)]


@pytest.mark.parametrize("name,D,symmetric,lazy", CASES_OBJ)
def test_objectives_within_the_error_bound(name, D, symmetric, lazy):
    """Per element against the float64 torch expression on the stored X (or on the rows regenerated from the same draw for the
    lazy population).  Worst measured ratio error / bound is printed."""
    o = obj(name)
    n = 256
    mu, sg = params(D, scale=2.0 if name != "ackley_twin" else 0.5)
    kw = dict(n_rows=n, symmetric=symmetric, seed=77 + D, stream_id=1)
    X, f = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
    ops.sample_eval(o.evok_objective_id, X, mu, sg, f=f, **kw)
    if lazy:
        ops.sample_eval(o.evok_objective_id, None, mu, sg, f=f, **kw)  # same draw, nothing stored: X above is its regeneration
    fe = ops.evaluate(o.evok_objective_id, X)
    torch.cuda.synchronize()
    for got in (f, fe):
        ok, ratio = _check_bound(name, X, got)
        print(f"{name} D={D} sym={symmetric} lazy={lazy}: worst error / bound {ratio:.3f}")
        assert ok, ratio


@pytest.mark.parametrize("mutation", ["column_off_by_one", "dropped_sum", "minus_row_on_plus_row", "D_off_by_one"])
def test_mutated_references_fall_outside_the_bound(mutation):
    failures = 0
    for name, D in itertools.product(SPECS, (3, 64, 1000)):
        o = obj(name)
        n = 128
        mu, sg = params(D, scale=2.0 if name != "ackley_twin" else 0.5)
        X, f = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
        ops.sample_eval(o.evok_objective_id, X, mu, sg, n_rows=n, symmetric=True, seed=9, stream_id=2, f=f)
        if mutation == "column_off_by_one":
            ok, _ = _check_bound(name, X, f, shift_j=1)
        elif mutation == "dropped_sum":
            ok, _ = _check_bound(name, X, f, drop=list(SPECS[name][0])[-1])
        elif mutation == "minus_row_on_plus_row":
            ok, _ = _check_bound(name, X, f.view(-1, 2).flip(1).reshape(-1))
        else:
            ok, _ = _check_bound(name, X, f, D_value=D + 1)
        failures += not ok
    assert failures >= 1


# ------------------------------------------------------------------------------------------------ NaN / inf
def test_nan_and_inf_reach_the_fitness_and_rank_as_before():
    o = FusedObjective("log_and_inverse", {"a": "log(x)", "b": "1 / x"}, "a + b")
    D, n = 8, 64
    mu = torch.linspace(-1.0, 1.0, D, device=DEV)
    sg = torch.full((D,), 0.5, device=DEV)
    X, f = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
    ops.sample_eval(o.evok_objective_id, X, mu, sg, n_rows=n, symmetric=True, seed=1, stream_id=0, f=f)
    torch.cuda.synchronize()
    assert torch.equal(torch.isnan(f), torch.isnan(o._torch_fn(X.double())))  # log of a negative sample: NaN, from the sampler
    X[3].zero_()  # 1 / 0 = inf, log(0) = -inf: -inf + inf = NaN
    X[5] = 2.0
    X[5, 0] = 0.0  # log(0) + 1/0 with the other columns finite: NaN too
    X[7] = torch.rand(D, device=DEV) + 0.5  # finite
    fe = ops.evaluate(o.evok_objective_id, X)
    ref = o._torch_fn(X.double())
    torch.cuda.synchronize()
    assert torch.equal(torch.isnan(fe), torch.isnan(ref)) and torch.equal(torch.isinf(fe), torch.isinf(ref))
    assert bool(torch.isnan(f).any()) and bool(torch.isnan(fe).any()) and bool(torch.isfinite(fe).any())
    for hib in (False, True):
        perm = torch.empty(n, dtype=torch.int64, device=DEV)
        ops.rank(fe, "centered", hib, perm=perm)
        assert torch.equal(perm.cpu(), torch.argsort(fe.cpu(), descending=not hib, stable=True))


# ------------------------------------------------------------------------------------------------ CUDA graphs, checkpoints
def test_graph_captured_as_the_first_generation_of_a_fresh_objective():
    """No eager launch of the objective before the capture: its module is loaded by the first call, which runs under capture."""
    o = FusedObjective("fresh_for_graph", {"s": "x**2 + 0.0078125*x"}, "s + D")
    oid = o.evok_objective_id
    D, n = 257, 512
    mu, sg = params(D)
    X, f = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with nat.private_workspaces(), torch.cuda.graph(graph):
        ops.sample_eval(oid, X, mu, sg, n_rows=n, symmetric=True, seed=4, stream_id=100, f=f, stream_offset=counter)
        counter.add_(1)
    for k in range(3):
        graph.replay()
        Xe, fe = torch.empty_like(X), torch.empty_like(f)
        ops.sample_eval(oid, Xe, mu, sg, n_rows=n, symmetric=True, seed=4, stream_id=100 + k, f=fe)
        torch.cuda.synchronize()
        assert same(X, Xe) and same(f, fe), k


@pytest.mark.parametrize("graph", [False, True])
def test_searcher_graph_replay_on_a_fresh_objective_equals_eager(graph):
    def run(objective, use_graph):
        s = PGPE(_problem(objective, 96), popsize=100, center_learning_rate=0.3, stdev_learning_rate=0.1, stdev_init=1.0)
        if use_graph:
            s.enable_cuda_graph()
        s.run(7)
        return s._distribution.mu.clone()

    fresh = FusedObjective(f"fresh_searcher_{graph}", {"s": f"x**2 + {0.25 + graph}*x"}, "s")
    a = run(fresh, graph)
    b = run(FusedObjective(f"fresh_searcher_{graph}", {"s": f"x**2 + {0.25 + graph}*x"}, "s"), False)
    assert same(a, b)


@pytest.mark.parametrize("lazy", [False, True])
def test_checkpoint_resume_is_bit_identical(lazy, tmp_path):
    from evotorch_b200.logging import PicklingLogger

    st = obj("styblinski_tang")

    def make():
        return CMAES(_problem(st, 150, lazy=lazy), stdev_init=1.0, popsize=200, separable=True)

    straight = make()
    straight.run(11)
    s = make()
    logger = PicklingLogger(s, interval=5, directory=str(tmp_path), prefix="st", verbose=False, checkpoint=True)
    s.run(5)
    resumed = PicklingLogger.resume(logger.last_file_name)
    assert resumed.problem._objective_func.evok_objective_id == st.evok_objective_id
    resumed.run(6)
    assert same(resumed.m, straight.m) and same(resumed.population.evals, straight.population.evals)
    assert len(pickle.dumps(st)) < 1000


# ------------------------------------------------------------------------------------------------ peer exchange
def _sim_world():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_peer_exchange_world.py")
    spec = importlib.util.spec_from_file_location("_peer_exchange_world", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("world_size", [2, 3])
def test_push_variant_at_simulated_world_sizes(world_size, symmetric, lazy):
    pw = _sim_world()
    o = obj("rastrigin_twin")
    D, N = 37, 3000
    counts = pw.shard_rows(N, world_size, 0, symmetric)[2]
    world = pw.SimWorld(counts, D)
    mu, sg = params(D)
    seed, sid = 0x1234_5678, 7
    world.poison()
    for r, px in enumerate(world.px):
        with world.on(r):
            Xr = None if lazy else torch.empty(counts[r], D, device=DEV)
            ops.sample_eval_push(o.evok_objective_id, Xr, mu, sg, n_rows=counts[r], symmetric=symmetric, seed=seed, stream_id=sid,
                                 row0=world.row0[r], peer=px)
    world.producers_done()
    for r, px in enumerate(world.px):
        with world.on(r):
            px.wait_fitness()
    world.check(1, 0)
    f = torch.empty(N, device=DEV)
    ops.sample_eval(o.evok_objective_id, None, mu, sg, n_rows=N, symmetric=symmetric, seed=seed, stream_id=sid, f=f)
    torch.cuda.synchronize()
    for r, px in enumerate(world.px):
        assert same(px.f_all, f), r


# ------------------------------------------------------------------------------------------------ errors
def test_cubin_missing_a_kernel_returns_the_error_and_launches_nothing():
    c = jit.compile_source(jit.ObjectiveSpec({"s": "x**2 + 0.5"}, "s").source)
    names = list(c.names)
    names[20] = "evok_no_such_kernel"
    oid = jit.register(c.cubin, names)
    D, n = 8, 16
    mu, sg = params(D)
    f = torch.full((n,), -1.0, device=DEV)
    X = torch.empty(n, D, device=DEV)
    torch.cuda.synchronize()
    before = ops.launch_count()
    lib = nat.lib()
    st = torch.cuda.current_stream().cuda_stream
    assert lib.evok_objective_load(oid) == E_NOKERNEL
    assert lib.evok_sample_eval(oid, X.data_ptr(), D, mu.data_ptr(), sg.data_ptr(), 0, n, D, 1, 0, 0, None, f.data_ptr(), st) == E_NOKERNEL
    assert lib.evok_eval(oid, X.data_ptr(), D, n, D, f.data_ptr(), st) == E_NOKERNEL
    with pytest.raises(ValueError, match="lacks"):
        ops.sample_eval(oid, None, mu, sg, n_rows=n, symmetric=True, seed=0, stream_id=0, f=f)
    torch.cuda.synchronize()
    assert ops.launch_count() == before and bool((f == -1.0).all())
    assert oid >= ops.OBJ_USER_BASE
