"""FusedObjective with pair terms on the GPU: every column layout of the sampling and evaluation kernels against the float64 torch
expression (per element, within an error bound), and bit-identity anchors between the kernels and through every fused path."""

import ast
import importlib.util
import itertools
import math
import os
import pickle

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, ops
    from evotorch_b200.algorithms import CEM, CMAES, PGPE, SNES
    from evotorch_b200.objectives import FusedObjective

DEV = "cuda"
U = 2.0**-24
C_BOUND = 1.0  # the constant of the error bound of tests/test_fused_objective_gpu.py
# 1 .. 8: one partial warp step; 127 .. 132 and 255 .. 260: the lane 31 -> lane 0 carry and partial groups; 256 columns: one
# unrolled sampler step; 512 / 516: the 4-group eval step; the rest: several steps with ragged tails
DIMS = [1, 2, 3, 4, 5, 8, 127, 128, 129, 132, 255, 256, 257, 260, 512, 516, 1000, 1028, 4096, 10_000, 10_001]


def _load(filename):
    """A sibling test module, by path (the tests directory is not a package)."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), filename)
    spec = importlib.util.spec_from_file_location("_" + filename[:-3], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


PAIR_SPECS = _load("test_pair_objective.py").PAIR_SPECS


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


_objs = {}


def obj(name):
    if name not in _objs:
        _objs[name] = FusedObjective(name, *PAIR_SPECS[name])
    return _objs[name]


def params(D, offset=False, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + D)
    mu = ((torch.rand(D + 1, generator=g) * 4 - 2) * scale).to(DEV)
    sg = (torch.rand(D + 1, generator=g) + 0.5).to(DEV)
    # offset: one float into the allocation, so the vectorised path is not taken even when D % 4 == 0
    return (mu[1:], sg[1:]) if offset else (mu[:D].clone(), sg[:D].clone())


# ------------------------------------------------------------------------------------------------ the float64 bound
def _err(node, env):
    """(value, error bound in units of 2^-24) of a parsed expression, in float64, first order."""
    if isinstance(node, ast.Expression):
        return _err(node.body, env)
    if isinstance(node, ast.Constant):
        v = torch.as_tensor(float(node.value), dtype=torch.float64, device=DEV)
        return v, v.abs()
    if isinstance(node, ast.Name):
        if node.id in ("pi", "e"):
            v = torch.as_tensor(getattr(math, node.id), dtype=torch.float64, device=DEV)
            return v, v.abs()
        return env[node.id]
    if isinstance(node, ast.UnaryOp):
        v, e = _err(node.operand, env)
        return (-v if isinstance(node.op, ast.USub) else v), e
    if isinstance(node, ast.BinOp):
        a, ea = _err(node.left, env)
        if isinstance(node.op, ast.Pow):
            n = int(node.right.value)  # the specs use positive integer exponents only
            v = a**n
            return v, n * (a.abs() ** (n - 1)) * ea + (n - 1) * v.abs()
        b, eb = _err(node.right, env)
        if isinstance(node.op, (ast.Add, ast.Sub)):
            v = a + b if isinstance(node.op, ast.Add) else a - b
            return v, ea + eb + v.abs()
        if isinstance(node.op, ast.Mult):
            v = a * b
            return v, ea * b.abs() + eb * a.abs() + v.abs()
        v = a / b
        return v, ea / b.abs() + eb * (a / (b * b)).abs() + v.abs()
    if isinstance(node, ast.Call):
        fn = node.func.id
        if fn in ("maximum", "minimum"):  # exact: the error of the operand chosen
            (a, ea), (b, eb) = _err(node.args[0], env), _err(node.args[1], env)
            a, b = torch.broadcast_tensors(a, b)
            pick = (a >= b) if fn == "maximum" else (a <= b)
            return torch.where(pick, a, b), torch.where(pick, ea, eb)
        a, ea = _err(node.args[0], env)
        f, d = {"sqrt": (torch.sqrt, lambda a: 0.5 / torch.sqrt(a)), "cos": (torch.cos, torch.sin),
                "abs": (torch.abs, lambda a: torch.ones_like(a))}[fn]
        v = f(a)
        return v, d(a).abs() * ea + 2 * v.abs()
    raise AssertionError(node)


def reference_and_bound(name, X, mutation=None):
    """float64 f and its error bound for the rows X (float32 values).  A pair term sees x = X[:, :-1] and xn = X[:, 1:] (both
    exact inputs) at j = 0 .. D-2.  `mutation` restates the reference wrongly, for the test of the bound's power:
      dropped_pair                 one pair (across the lane 0 -> lane 1 boundary where there is one) left out;
      wrap_around_pair             the pair (x_{D-1}, x_0) added at j = D-1;
      j_shifted                    j + 1 in the pair terms;
      plus_neighbour_on_minus_row  the - row's pairs take xn from its + row (symmetric sampling: rows 2u, 2u + 1)."""
    sums, value = PAIR_SPECS[name]
    X = X.double()
    n, D = X.shape
    k_eff = math.ceil(D / 32) + 5  # per-lane sums, then five shuffle rounds
    S, eS = {}, {}
    for s, t in sums.items():
        tree = ast.parse(t, mode="eval")
        if any(isinstance(nd, ast.Name) and nd.id == "xn" for nd in ast.walk(tree)):
            x, xn = X[:, :-1], X[:, 1:]
            j = torch.arange(D - 1, dtype=torch.float64, device=DEV)
            if mutation == "dropped_pair" and D >= 2:
                keep = torch.ones(D - 1, dtype=torch.bool, device=DEV)
                keep[min(3, D - 2)] = False
                x, xn, j = x[:, keep], xn[:, keep], j[keep]
            elif mutation == "wrap_around_pair":
                x, xn = torch.cat([x, X[:, -1:]], 1), torch.cat([xn, X[:, :1]], 1)
                j = torch.arange(D, dtype=torch.float64, device=DEV)
            elif mutation == "j_shifted":
                j = j + 1
            elif mutation == "plus_neighbour_on_minus_row":
                xn = xn.clone()
                xn[1::2] = X[0::2, 1:]
        else:
            x, xn, j = X, None, torch.arange(D, dtype=torch.float64, device=DEV)
        zero = torch.zeros_like(x)
        env = {"x": (x, zero), "j": (j.expand_as(x), zero), "D": (torch.full_like(x, float(D)), zero)}
        if xn is not None:
            env["xn"] = (xn, zero)
        v, e = _err(tree, env)
        v, e = torch.broadcast_to(v, x.shape), torch.broadcast_to(e, x.shape)
        S[s] = v.sum(1)
        eS[s] = e.sum(1) + k_eff * v.abs().sum(1)
    tree = ast.parse(value, mode="eval")
    base = {s: (S[s], torch.zeros_like(S[s])) for s in S}
    base["D"] = (torch.full((n,), float(D), dtype=torch.float64, device=DEV), torch.zeros(n, dtype=torch.float64, device=DEV))
    f, e_value = _err(tree, base)
    # the sums' errors carried through `value` at the corners of their intervals
    carried = torch.zeros_like(f)
    for signs in itertools.product((-1.0, 1.0), repeat=len(S)):
        corner = {s: (S[s] + sg * C_BOUND * U * eS[s], torch.zeros_like(S[s])) for s, sg in zip(S, signs)}
        corner["D"] = base["D"]
        carried = torch.maximum(carried, (_err(tree, corner)[0] - f).abs())
    return f, C_BOUND * U * e_value + carried


def within_bound(name, X, f, mutation=None):
    ref, bound = reference_and_bound(name, X, mutation)
    err = (f.double() - ref).abs()
    return bool((err <= bound).all()), float((err / bound.clamp_min(1e-300)).max())


# ------------------------------------------------------------------------------------------------ column layouts
@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("D", DIMS)
def test_column_layouts_within_the_float64_bound(D, symmetric, offset):
    """Every instantiation at every layout: stored and lazy sampling (and the SQ sampler), evaluation of the stored X on its own
    path and on the scalar path.  X and q are the built-in sampler's bit for bit, lazy fitnesses the stored ones, and on the
    vectorised path evaluation reproduces the sampler's fitnesses bit for bit (one pair-ownership rule in both kernels)."""
    n = 2 * 37
    mu, sg = params(D, offset)
    kw = dict(n_rows=n, symmetric=symmetric, seed=0x5EED0 + D, stream_id=3, row0=4)
    vec = D % 4 == 0 and not offset
    Xb = torch.empty(n, D, device=DEV)
    ops.sample_eval(ops.OBJ_SPHERE, Xb, mu, sg, f=torch.empty(n, device=DEV), **kw)
    if not symmetric:
        qb = torch.empty(n, device=DEV)
        ops.sample_eval_sq(ops.OBJ_SPHERE, None, mu, sg, qb, f=torch.empty(n, device=DEV), **{k: v for k, v in kw.items() if k != "symmetric"})
    for name in PAIR_SPECS:
        oid = obj(name).evok_objective_id
        X, f, fl = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        ops.sample_eval(oid, X, mu, sg, f=f, **kw)
        ops.sample_eval(oid, None, mu, sg, f=fl, **kw)
        fe = ops.evaluate(oid, X)
        fe_odd = ops.evaluate(oid, torch.empty(n, D + 1, device=DEV)[:, 1:].copy_(X))  # the scalar evaluation path
        if not symmetric:
            kq = {k: v for k, v in kw.items() if k != "symmetric"}
            Xq, fq, q, flq, ql = (torch.empty(n, D, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV),
                                  torch.empty(n, device=DEV), torch.empty(n, device=DEV))
            ops.sample_eval_sq(oid, Xq, mu, sg, q, f=fq, **kq)
            ops.sample_eval_sq(oid, None, mu, sg, ql, f=flq, **kq)
        torch.cuda.synchronize()
        assert same(X, Xb), name
        assert same(fl, f), name
        if vec:
            assert same(fe, f), name
        if not symmetric:
            assert same(Xq, X) and same(fq, f) and same(flq, f) and same(q, qb) and same(ql, qb), name
        for label, got in (("sampler", f), ("eval", fe), ("scalar eval", fe_odd)):
            ok, ratio = within_bound(name, X, got)
            print(f"{name} D={D} sym={symmetric} offset={offset} {label}: worst error / bound {ratio:.3f}")
            assert ok, (name, label, ratio)


@pytest.mark.parametrize("mutation", ["dropped_pair", "wrap_around_pair", "j_shifted", "plus_neighbour_on_minus_row"])
def test_mutated_references_fall_outside_the_bound(mutation):
    failures, cases = 0, 0
    for name, D in itertools.product(PAIR_SPECS, (3, 64, 129, 1000)):
        o = obj(name)
        n = 128
        mu, sg = params(D)
        X, f = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
        ops.sample_eval(o.evok_objective_id, X, mu, sg, n_rows=n, symmetric=True, seed=9, stream_id=2, f=f)
        torch.cuda.synchronize()
        assert within_bound(name, X, f)[0], name  # the true reference holds
        failures += not within_bound(name, X, f, mutation)[0]
        cases += 1
    print(f"{mutation}: outside the bound in {failures} of {cases} cases")
    assert failures >= 1


# ------------------------------------------------------------------------------------------------ whole searchers
def _problem(objective, D, lazy=False, seed=3):
    return Problem("min", objective, initial_bounds=(-2, 2), solution_length=D, device=DEV, seed=seed, lazy_population=lazy)


SEARCHERS = {
    "pgpe": lambda p: PGPE(p, popsize=200, center_learning_rate=0.3, stdev_learning_rate=0.1, stdev_init=1.0),
    "snes": lambda p: SNES(p, popsize=120, stdev_init=1.0),
    "cem": lambda p: CEM(p, popsize=120, parenthood_ratio=0.5, stdev_init=1.0),
    # a given centre: a materialised CMA-ES draws an initial population before a random centre, a lazy one does not
    "sepcma": lambda p: CMAES(p, stdev_init=1.0, popsize=150, separable=True, center_init=_centre(p)),
    # a Cholesky every generation: capturable
    "cmaes": lambda p: CMAES(p, stdev_init=1.0, popsize=64, limit_C_decomposition=False, center_init=_centre(p)),
}
# (lazy, graph) runs that give the same trajectory bit for bit.  PGPE's lazy gradient regenerates the + rows and sums them in
# another order than the materialised one, so its lazy runs form their own group, equal to the materialised runs in the first
# generation (the same draw from the same distribution) and bounded against float64 in every generation.
GROUPS = {"pgpe": [[(False, False), (False, True)], [(True, False), (True, True)]], "snes": [[(False, False), (False, True)]],
          "cem": [[(False, False), (False, True)]], "sepcma": [[(False, False), (True, False), (False, True), (True, True)]],
          "cmaes": [[(False, False), (False, True)]]}
SEARCHER_CASES = [(name, D) for name in SEARCHERS for D in ((37, 40) if name == "cmaes" else (130, 260))]


def _centre(p):
    return torch.linspace(-1.5, 1.5, p.solution_length, device=DEV)


def _state(s):
    if isinstance(s, CMAES):
        return [s.m, s.sigma.reshape(-1)] + ([s.C] if hasattr(s, "C") else [])
    d = s._distribution
    return [d.mu, d.sigma]


@pytest.mark.parametrize("name,D", SEARCHER_CASES)
def test_searchers_lazy_and_graph_replay_bit_identical_and_within_the_bound(name, D):
    """Rosenbrock, 6 generations of every (lazy, graph) run of a group: the same trajectory bit for bit, and every generation's
    fitnesses within the float64 bound on the population evaluated (regenerated from its Philox record when lazy)."""
    o = obj("rosenbrock")

    def run(lazy, graph):
        s = SEARCHERS[name](_problem(o, D, lazy=lazy))
        if graph:
            s.enable_cuda_graph()
        hist = []
        for g in range(6):
            s.step()
            X, f = s.population.values.clone(), s.population.evals.clone()
            hist.append([t.detach().clone() for t in _state(s)] + [f, X])
            ok, ratio = within_bound("rosenbrock", X, f[:, 0])
            assert ok, (lazy, graph, g, ratio)
        torch.cuda.synchronize()
        if graph:
            assert s._graph is not None, "the generation was not captured"
        return hist

    firsts = []
    for group in GROUPS[name]:
        ref = run(*group[0])
        firsts.append(ref[0][-2:])
        for lazy, graph in group[1:]:
            other = run(lazy, graph)
            for g, (a, b) in enumerate(zip(ref, other)):
                for x, y in zip(a, b):
                    assert same(x, y), f"{group[0]} against lazy={lazy} graph={graph}: generation {g}"
    for f, X in firsts[1:]:
        assert same(f, firsts[0][0]) and same(X, firsts[0][1])


@pytest.mark.parametrize("lazy", [False, True])
def test_checkpoint_resume_is_bit_identical(lazy, tmp_path):
    from evotorch_b200.logging import PicklingLogger

    o = obj("dixon_price")

    def make():
        return CMAES(_problem(o, 150, lazy=lazy), stdev_init=1.0, popsize=200, separable=True)

    straight = make()
    straight.run(11)
    s = make()
    logger = PicklingLogger(s, interval=5, directory=str(tmp_path), prefix="dp", verbose=False, checkpoint=True)
    s.run(5)
    resumed = PicklingLogger.resume(logger.last_file_name)
    assert resumed.problem._objective_func.evok_objective_id == o.evok_objective_id
    resumed.run(6)
    assert same(resumed.m, straight.m) and same(resumed.population.evals, straight.population.evals)
    assert len(pickle.dumps(o)) < 1000


# ------------------------------------------------------------------------------------------------ peer exchange
# uneven shards (a symmetric layout keeps whole +/- pairs on one rank)
SHARDS = {(2, True): [1000, 2002], (2, False): [1001, 1999], (3, True): [600, 1402, 1000], (3, False): [701, 1300, 1001]}


@pytest.mark.parametrize("D", [257, 260])
@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("world_size", [2, 3])
def test_push_variant_at_simulated_world_sizes(world_size, symmetric, lazy, D):
    pw = _load("test_peer_exchange_world.py")
    o = obj("mix4")
    counts = SHARDS[(world_size, symmetric)]
    N = sum(counts)
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
    X, f = torch.empty(N, D, device=DEV), torch.empty(N, device=DEV)
    ops.sample_eval(o.evok_objective_id, X, mu, sg, n_rows=N, symmetric=symmetric, seed=seed, stream_id=sid, f=f)
    torch.cuda.synchronize()
    for r, px in enumerate(world.px):
        assert same(px.f_all, f), r
    assert within_bound("mix4", X, f)[0]


# ------------------------------------------------------------------------------------------------ NaN / inf
def test_nan_and_inf_in_a_pair_term_reach_the_fitness():
    lg = FusedObjective("pair_log_inverse", {"a": "log(xn - x)", "b": "1 / (xn - x)"}, "a + b")
    pr = FusedObjective("pair_product", {"s": "x * xn"}, "s")
    D, n = 8, 64
    mu = torch.linspace(-1.0, 1.0, D, device=DEV)
    sg = torch.full((D,), 0.5, device=DEV)
    X, f = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
    ops.sample_eval(lg.evok_objective_id, X, mu, sg, n_rows=n, symmetric=True, seed=1, stream_id=0, f=f)
    torch.cuda.synchronize()
    ref = lg._torch_fn(X.double())
    assert torch.equal(torch.isnan(f), torch.isnan(ref)) and bool(torch.isnan(f).any()) and bool(torch.isfinite(f).any())
    X[3] = 1.0  # xn - x = 0: log 0 + 1/0 = -inf + inf = NaN
    X[5] = torch.arange(D, dtype=torch.float32, device=DEV)  # log 1 + 1 per pair: finite
    X[6] = torch.arange(D, dtype=torch.float32, device=DEV)
    X[6, 7] = float("inf")  # log(inf) + 1/inf = inf in the last pair only
    for Xv in (X, torch.empty(n, D + 1, device=DEV)[:, 1:].copy_(X)):  # the vectorised and the scalar evaluation
        fe = ops.evaluate(lg.evok_objective_id, Xv)
        torch.cuda.synchronize()
        ref = lg._torch_fn(X.double())
        assert torch.equal(torch.isnan(fe), torch.isnan(ref)) and torch.equal(torch.isinf(fe), torch.isinf(ref))
        assert bool(torch.isnan(fe[3])) and bool(torch.isfinite(fe[5])) and float(fe[6]) == math.inf
    # an infinite mean: column 3 is +inf in every row, so x_2 * x_3 and x_3 * x_4 are infinite with the signs of x_2 and x_4
    mu_inf = mu.clone()
    mu_inf[3] = math.inf
    for symmetric in (True, False):
        ops.sample_eval(pr.evok_objective_id, X, mu_inf, sg, n_rows=n, symmetric=symmetric, seed=2, stream_id=0, f=f)
        torch.cuda.synchronize()
        ref = pr._torch_fn(X.double())
        assert torch.equal(torch.isnan(f), torch.isnan(ref)) and torch.equal(f.double()[torch.isinf(ref)], ref[torch.isinf(ref)])
        assert bool(torch.isnan(f).any()) and bool((f == math.inf).any()) and bool((f == -math.inf).any())
