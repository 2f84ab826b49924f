"""Batched sample-and-evaluate (evok_sample_eval_batched) and the batched rebuild gradient (evok_grad_batched_regen) on the GPU, and
the functional ask / tell runs built on them (pgpe_ask_and_evaluate / cem_ask_and_evaluate, materialised or lazy).

- Sampler bits: per probed item, X and f equal evok_sample_eval(stream_id0 + b) bit for bit, X equals evok_sample_batched, and on the
  vectorised path f equals evok_eval of the stored rows; the element and pair specs are also checked against the float64 bound of
  tests/test_pair_objective_gpu.py (the built-in Rastrigin and Ackley use fast intrinsics: their accuracy is the single-search
  sampler's, which these tests reproduce bit for bit).
- Gradient bits: grad_batched_regen equals grad_batched over the stored population bit for bit, and lies within the float64 bound of
  tests/test_functional_batched.py against oracle/functional_oracle.py.
- Whole runs: 10 generations materialised, lazy, and ask + ops.evaluate + tell are the same trajectory bit for bit.
"""

import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import ops
    from evotorch_b200.algorithms import functional as F
    from evotorch_b200.objectives import FusedObjective, ackley, rastrigin, sphere

from oracle import functional_oracle as FO

DEV = "cuda"
BIG = 70000  # more items than one launch's grid y holds (65535)
ELEMENT = {"styblinski_tang": ({"s": "x**4 - 16*x**2 + 5*x"}, "0.5 * s"), "sphere_spec": ({"s": "x**2"}, "s")}


def _load(filename):
    """A sibling test module, by path (the tests directory is not a package)."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), filename)
    spec = importlib.util.spec_from_file_location("_ff_" + filename[:-3], path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


PG = _load("test_pair_objective_gpu.py")  # the float64 bound of the fused objectives
PG.PAIR_SPECS.update(ELEMENT)
FB = _load("test_functional_batched.py")  # the float64 bound of the batched stages

_objs = {}


def objective(name):
    if name not in _objs:
        if name in ("sphere", "rastrigin", "ackley"):
            _objs[name] = {"sphere": sphere, "rastrigin": rastrigin, "ackley": ackley}[name]
        else:
            _objs[name] = FusedObjective(name, *PG.PAIR_SPECS[name])
            _objs[name].compile_batched()
    return _objs[name]


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def operands(B, D, layout, seed=0):
    """(mu, sigma) as the batched call takes them and per item: shared (D,), per item (B, D), or a 4-byte offset per-item mu."""
    g = torch.Generator().manual_seed(seed + D + B)
    mu = (torch.rand(B * D + 1, generator=g) * 4 - 2).to(DEV)
    sg = (torch.rand(B, D, generator=g) + 0.5).to(DEV)
    if layout == "shared":
        return mu[:D].clone(), sg[0].clone()
    if layout == "offset":  # one float into the allocation: every item's mu is misaligned, so the vectorised path is not taken
        return mu[1:].view(B, D), sg
    return mu[:B * D].view(B, D).clone(), sg


def item(t, b):
    return t if t.ndim == 1 else t[b]


OBJECTIVES = ["sphere", "rastrigin", "ackley", "styblinski_tang", "rosenbrock"]


@pytest.mark.parametrize("name", OBJECTIVES)
@pytest.mark.parametrize("symmetric", [False, True])
@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("D", [64, 63, 1])
@pytest.mark.parametrize("layout", ["shared", "per_item", "offset"])
def test_sampler_bits_per_item(name, symmetric, lazy, D, layout):
    o = objective(name)
    oid = o.evok_objective_id
    B, n = 3, 10
    mu, sg = operands(B, D, layout)
    seed, sid0 = 0xC0FFEE + D, 5
    X = None if lazy else torch.empty(B, n, D, device=DEV)
    f = torch.full((B, n), float("nan"), device=DEV)
    ops.sample_eval_batched(oid, X, mu, sg, f, symmetric=symmetric, seed=seed, stream_id0=sid0)
    Xs = torch.empty(B, n, D, device=DEV)
    ops.sample_batched(Xs, mu, sg, symmetric=symmetric, seed=seed, stream_id0=sid0)
    if X is not None:
        assert same(X, Xs)
    vec = D % 4 == 0 and layout != "offset"
    for b in range(B):
        Xb, fb = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
        m, s = item(mu, b).contiguous() if layout != "offset" else item(mu, b), item(sg, b).contiguous()
        ops.sample_eval(oid, Xb, m, s, n_rows=n, symmetric=symmetric, seed=seed, stream_id=sid0 + b, f=fb)
        assert same(Xs[b], Xb), b
        assert same(f[b], fb), b
        if vec:
            assert same(f[b], ops.evaluate(oid, Xs[b].contiguous())), b
        spec = {"sphere": "sphere_spec"}.get(name, name)  # the built-in sphere folds fmaf(x, x, s): the bound of the spec x**2
        if spec in PG.PAIR_SPECS:
            ok, worst = PG.within_bound(spec, Xs[b], f[b])
            assert ok, (b, worst)


@pytest.mark.parametrize("name", OBJECTIVES)
@pytest.mark.parametrize("lazy", [False, True])
def test_sampler_bits_across_the_item_chunks(name, lazy):
    """70 000 items at small N and D: the first, last and boundary items of the 65535-item chunks follow their own streams."""
    o = objective(name)
    oid = o.evok_objective_id
    B, n, D = BIG, 2, 8
    mu, sg = operands(B, D, "per_item", seed=1)
    X = None if lazy else torch.empty(B, n, D, device=DEV)
    f = torch.empty(B, n, device=DEV)
    ops.sample_eval_batched(oid, X, mu, sg, f, symmetric=True, seed=77, stream_id0=3)
    for b in (0, 1, 65534, 65535, 65536, B - 1):
        Xb, fb = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
        ops.sample_eval(oid, Xb, mu[b].contiguous(), sg[b].contiguous(), n_rows=n, symmetric=True, seed=77, stream_id=3 + b, f=fb)
        assert same(f[b], fb), b
        if X is not None:
            assert same(X[b], Xb), b


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
@pytest.mark.parametrize("D", [64, 63])
def test_an_item_reads_only_its_own_centre(name, D):
    """Items 0 and 2 have NaN centres and stdevs: item 1 (non-zero item stride) must not see them."""
    oid = objective(name).evok_objective_id
    B, n = 3, 8
    mu, sg = operands(B, D, "per_item", seed=2)
    mu[0], mu[2], sg[0], sg[2] = float("nan"), float("nan"), float("nan"), float("nan")
    X, f = torch.empty(B, n, D, device=DEV), torch.empty(B, n, device=DEV)
    ops.sample_eval_batched(oid, X, mu, sg, f, symmetric=False, seed=9, stream_id0=0)
    Xb, fb = torch.empty(n, D, device=DEV), torch.empty(n, device=DEV)
    ops.sample_eval(oid, Xb, mu[1].contiguous(), sg[1].contiguous(), n_rows=n, symmetric=False, seed=9, stream_id=1, f=fb)
    assert torch.isfinite(f[1]).all() and torch.isfinite(X[1]).all()
    assert same(f[1], fb) and same(X[1], Xb)
    assert torch.isnan(f[0]).all() and torch.isnan(f[2]).all()


def test_registered_id_without_batched_kernels_launches_nothing():
    o = FusedObjective("no_batched_kernels", {"s": "x**2 + 0.5*x"}, "s")
    before = ops.launch_count()
    with pytest.raises(ValueError, match="code -7"):
        ops.sample_eval_batched(o.evok_objective_id, None, torch.zeros(8, device=DEV), torch.ones(8, device=DEV),
                                torch.empty(2, 4, device=DEV), symmetric=False, seed=0)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------ K4 rebuild
@pytest.mark.parametrize("form", [0, 1, 2, 3])
@pytest.mark.parametrize("D", [64, 63])
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("B,n", [(1, 64), (3, 200), (BIG, 4)])
def test_grad_batched_regen_equals_grad_batched(form, D, shared, B, n):
    if B == BIG and D == 63 and not shared:
        pytest.skip("one 70 000-item layout per form and D is enough")
    sym = form == 1  # GRAD_SYMMETRIC: the + rows of a symmetric population
    mu, sg = operands(B, D, "shared" if shared else "per_item", seed=form)
    seed, sid0 = 1234 + form, 11
    X = torch.empty(B, n, D, device=DEV)
    ops.sample_batched(X, mu, sg, symmetric=sym, seed=seed, stream_id0=sid0)
    g = torch.Generator().manual_seed(B + n + D)
    if form == ops.GRAD_MOMENTS:
        w = (torch.rand(B, n, generator=g) < 0.3).float()
    else:
        w = torch.randn(B, n, generator=g)
        w[torch.rand(B, n, generator=g) < 0.25] = 0.0  # rows that are skipped
    w = w.to(DEV)
    a = ops.grad_batched(form, X, w, mu, sg, 0.37, 1.9)
    r = ops.grad_batched_regen(form, w, mu, sg, 0.37, 1.9, seed=seed, stream_id0=sid0)
    assert same(a[0], r[0]) and same(a[1], r[1])
    # and within the float64 bound of the batched gradient against the oracle
    Xh, wh, muh, sgh = X.cpu().numpy(), w.cpu().numpy(), mu.cpu().numpy(), sg.cpu().numpy()
    k_eff = (n // 2 if sym else n) + 6
    probes = range(B) if B <= 5 else (0, 65534, 65535, B - 1)
    for b in probes:
        m, s = (muh, sgh) if shared else (muh[b], sgh[b])
        ref = FO.weighted_sums(form, Xh[b], wh[b], m, s)
        FB._check(f"s1 item {b}", r[0][b].cpu().numpy(), 0.37 * ref["s1"], FB.C_ROUND * FB.EPS32 * k_eff * 0.37 * ref["s1_mag"] + 1e-30)
        FB._check(f"s2 item {b}", r[1][b].cpu().numpy(), 1.9 * ref["s2"], FB.C_ROUND * FB.EPS32 * k_eff * 1.9 * ref["s2_mag"] + 1e-30)


@pytest.mark.parametrize("form", [0, 1, 2, 3])
@pytest.mark.parametrize("shared", [True, False])
def test_grad_batched_regen_equals_grad_batched_one_wide_item(form, shared):
    """One item at a shape where a single search would take the TMA kernel (D >= 512, at least 4096 row units): the batch keeps
    the LDG plan, so the stored and rebuilt populations still give the same bits."""
    test_grad_batched_regen_equals_grad_batched(form, 1024, shared, 1, 8192)


# ------------------------------------------------------------------------------------------------ whole runs
def _pgpe_state(batch, layout, opt, ranking, symmetric, D):
    g = torch.Generator().manual_seed(len(batch) * 7 + D)
    full = tuple(batch) + (D,)
    center = (torch.rand(full if layout != "shared_center" else (D,), generator=g) * 4 - 2).to(DEV)
    stdev = (torch.rand(full if layout == "shared_center" else (D,), generator=g) * 0.5 + 0.5).to(DEV)
    if layout == "both_batched":
        stdev = stdev.expand(full).clone()
    cfg = {"clipup": {}, "adam": {}, "sgd": {"momentum": 0.9}}[opt]
    return F.pgpe(center_init=center, center_learning_rate=0.2, stdev_learning_rate=0.1, stdev_init=stdev, objective_sense="min",
                  ranking_method=ranking, optimizer=opt, optimizer_config=cfg, symmetric=symmetric)


def _run_pgpe(state, mode, o, popsize, gens=10):
    torch.manual_seed(2024)
    out = []
    for _ in range(gens):
        if mode == "ask_evaluate":
            values = F.pgpe_ask(state, popsize=popsize)
            evals = ops.evaluate(o.evok_objective_id, values.view(-1, values.shape[-1])).view(values.shape[:-1])
        else:
            values, evals = F.pgpe_ask_and_evaluate(state, popsize=popsize, objective=o, lazy=(mode == "lazy"))
        state = F.pgpe_tell(state, values, evals)
        out.append((evals.clone(), state.optimizer_state.center.clone(), state.stdev.clone()))
    return out


def _same_runs(a, b):
    return all(same(x, y) for ga, gb in zip(a, b) for x, y in zip(ga, gb))


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
@pytest.mark.parametrize("opt", ["clipup", "adam", "sgd"])
@pytest.mark.parametrize("ranking", ["centered", "linear"])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("batch,layout", [((), "both_batched"), ((3,), "both_batched"), ((2, 3), "both_batched"), ((3,), "shared_center"),
                                          ((2, 3), "shared_stdev")])
def test_pgpe_runs_materialised_lazy_and_ask_evaluate_are_bit_identical(name, opt, ranking, symmetric, batch, layout):
    o = objective(name)
    D, popsize = 32, 12
    runs = {mode: _run_pgpe(_pgpe_state(batch, layout, opt, ranking, symmetric, D), mode, o, popsize)
            for mode in ("materialised", "lazy", "ask_evaluate")}
    assert _same_runs(runs["materialised"], runs["lazy"])
    assert _same_runs(runs["materialised"], runs["ask_evaluate"])
    assert runs["materialised"][0][0].shape == tuple(batch) + (popsize,)
    assert not same(runs["materialised"][0][1], runs["materialised"][-1][1])  # the search moved


def _run_cem(state, mode, o, popsize, gens=10):
    torch.manual_seed(99)
    out = []
    for _ in range(gens):
        if mode == "ask_evaluate":
            values = F.cem_ask(state, popsize=popsize)
            evals = ops.evaluate(o.evok_objective_id, values.view(-1, values.shape[-1])).view(values.shape[:-1])
        else:
            values, evals = F.cem_ask_and_evaluate(state, popsize=popsize, objective=o, lazy=(mode == "lazy"))
        state = F.cem_tell(state, values, evals)
        out.append((evals.clone(), state.center.clone(), state.stdev.clone()))
    return out


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
@pytest.mark.parametrize("batch,layout", [((), "both_batched"), ((3,), "both_batched"), ((2, 3), "both_batched"), ((3,), "shared_center"),
                                          ((2, 3), "shared_stdev")])
def test_cem_runs_materialised_lazy_and_ask_evaluate_are_bit_identical(name, batch, layout):
    o = objective(name)
    D, popsize = 32, 20

    def state():
        g = torch.Generator().manual_seed(len(batch) + D)
        full = tuple(batch) + (D,)
        center = (torch.rand(full if layout != "shared_center" else (D,), generator=g) * 4 - 2).to(DEV)
        stdev = (torch.rand(full if layout == "shared_center" else (D,), generator=g) * 0.5 + 0.5).to(DEV)
        return F.cem(center_init=center, stdev_init=stdev, parenthood_ratio=0.25, objective_sense="min", stdev_max_change=0.3)

    runs = {mode: _run_cem(state(), mode, o, popsize) for mode in ("materialised", "lazy", "ask_evaluate")}
    assert _same_runs(runs["materialised"], runs["lazy"])
    assert _same_runs(runs["materialised"], runs["ask_evaluate"])


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("swept", ["stdev_learning_rate", "stdev_max_change", "both"])
def test_pgpe_sweep_over_hyper_parameters_lazy_equals_materialised(name, symmetric, swept):
    """A sweep: batched stdev_learning_rate / stdev_max_change (3 items) over an unbatched centre and stdev.  The first ask draws one
    population, which the tell broadcasts to the 3 items; the lazy run must follow the materialised one bit for bit."""
    o = objective(name)
    D, popsize = 32, 12

    def state():
        g = torch.Generator().manual_seed(D)
        center = (torch.rand(D, generator=g) * 4 - 2).to(DEV)
        lr = torch.tensor([0.05, 0.1, 0.2]) if swept != "stdev_max_change" else 0.1
        mc = torch.tensor([0.1, 0.2, 0.3])[:, None].expand(3, D) if swept != "stdev_learning_rate" else 0.2
        return F.pgpe(center_init=center, center_learning_rate=0.2, stdev_learning_rate=lr, stdev_init=0.7, stdev_max_change=mc,
                      objective_sense="min", symmetric=symmetric)

    runs = {mode: _run_pgpe(state(), mode, o, popsize) for mode in ("materialised", "lazy", "ask_evaluate")}
    assert runs["materialised"][0][0].shape == (popsize,)  # the first population is not batched; the next ones are
    assert runs["materialised"][1][0].shape == (3, popsize)
    assert _same_runs(runs["materialised"], runs["lazy"])
    assert _same_runs(runs["materialised"], runs["ask_evaluate"])


@pytest.mark.parametrize("name", ["rastrigin", "rosenbrock"])
def test_cem_sweep_over_stdev_max_change_lazy_equals_materialised(name):
    o = objective(name)
    D, popsize = 32, 20

    def state():
        g = torch.Generator().manual_seed(D + 1)
        center = (torch.rand(D, generator=g) * 4 - 2).to(DEV)
        mc = torch.tensor([0.1, 0.2, 0.3])[:, None].expand(3, D)
        return F.cem(center_init=center, stdev_init=0.7, parenthood_ratio=0.25, objective_sense="min", stdev_max_change=mc)

    runs = {mode: _run_cem(state(), mode, o, popsize) for mode in ("materialised", "lazy", "ask_evaluate")}
    assert runs["materialised"][1][0].shape == (3, popsize)
    assert _same_runs(runs["materialised"], runs["lazy"])
    assert _same_runs(runs["materialised"], runs["ask_evaluate"])


def test_materialised_population_is_the_asked_one_and_lazy_materialises_it():
    state = _pgpe_state((3,), "both_batched", "clipup", "centered", True, 40)
    torch.manual_seed(5)
    X, f = F.pgpe_ask_and_evaluate(state, popsize=8, objective=rastrigin)
    torch.manual_seed(5)
    assert same(X, F.pgpe_ask(state, popsize=8))
    torch.manual_seed(5)
    pop, f2 = F.pgpe_ask_and_evaluate(state, popsize=8, objective=rastrigin, lazy=True)
    assert isinstance(pop, F.LazyPopulation) and pop.shape == X.shape
    assert same(pop.materialize(), X) and same(f2, f)


def test_lazy_population_told_to_another_state_raises():
    state = _pgpe_state((2,), "both_batched", "clipup", "centered", True, 16)
    pop, evals = F.pgpe_ask_and_evaluate(state, popsize=4, objective=rastrigin, lazy=True)
    other = _pgpe_state((2,), "both_batched", "clipup", "centered", True, 16)
    with pytest.raises(ValueError, match="another centre"):
        F.pgpe_tell(other, pop, evals)
    with pytest.raises(ValueError, match="symmetric"):
        F.pgpe_tell(state._replace(symmetric=False), pop, evals)
    new = F.pgpe_tell(state, pop, evals)
    with pytest.raises(ValueError, match="another"):
        F.pgpe_tell(new, pop, evals)  # the next state's centre is a new tensor
    state.stdev.mul_(1.0)  # an in-place change of the stdev it was drawn from
    with pytest.raises(ValueError, match="another stdev"):
        F.pgpe_tell(state, pop, evals)
    cstate = F.cem(center_init=torch.zeros(2, 16, device=DEV), stdev_init=1.0, parenthood_ratio=0.5, objective_sense="min")
    cpop, cev = F.cem_ask_and_evaluate(cstate, popsize=4, objective=rastrigin, lazy=True)
    with pytest.raises(ValueError, match="another"):
        F.cem_tell(cstate._replace(center=cstate.center.clone()), cpop, cev)


def test_lazy_run_memory_is_of_the_order_of_fitnesses_and_centres():
    """1024 searches x 1000 solutions x 1000 dimensions: the population would take 4.1 GB; the lazy generation allocates O(B N + B D)."""
    B, N, D = 1024, 1000, 1000
    state = F.pgpe(center_init=torch.zeros(B, D, device=DEV), center_learning_rate=0.2, stdev_learning_rate=0.1, stdev_init=1.0,
                   objective_sense="min")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    pop, evals = F.pgpe_ask_and_evaluate(state, popsize=N, objective=rastrigin, lazy=True)
    state = F.pgpe_tell(state, pop, evals)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= 16 * 4 * (B * N + B * D), peak
    assert torch.isfinite(state.optimizer_state.center).all()
