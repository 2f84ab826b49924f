"""The hybrid gradient pass (part of the population rows rebuilt from their Philox counters, the rest read from HBM) must give
exactly what the reading pass gives: at the kernel level for every split, and along whole searcher trajectories, eager and
replayed from a CUDA graph.  A population modified in place after sampling must be read, not rebuilt."""

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, ops
    from evotorch_b200.algorithms import PGPE, SNES
    from evotorch_b200.objectives import rastrigin

DEV = "cuda"
SEED, STREAM, ROW0 = 99, 7, 4096
# (rows, columns): one 1024-column tile with a 4-unit last row chunk; a ragged second column tile; ten column tiles of which
# the last is ragged; a ragged tile together with a short last row chunk and a short last row group
SHAPES = [(8192, 1024), (20000, 2000), (16384, 10000), (9000, 1536)]


def _forms():
    return {"symmetric": ops.GRAD_SYMMETRIC, "separable": ops.GRAD_SEPARABLE, "exp": ops.GRAD_EXP}


@pytest.mark.parametrize("offset", [False, True], ids=["no_offset", "stream_offset"])
@pytest.mark.parametrize("form_name", ["symmetric", "separable", "exp"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{n}x{d}" for n, d in SHAPES])
def test_hybrid_gradient_is_bit_identical_to_reading_every_row(shape, form_name, offset):
    n, d = shape
    form = _forms()[form_name]
    gen = torch.Generator(device=DEV).manual_seed(n + d)
    mu = torch.rand(d, generator=gen, device=DEV) * 4.0 - 2.0
    sigma = torch.rand(d, generator=gen, device=DEV) * 0.9 + 0.1
    off = torch.tensor([5], dtype=torch.int32, device=DEV) if offset else None
    X = torch.empty(n, d, device=DEV)
    ops.sample_eval(ops.OBJ_NONE, X, mu, sigma, n_rows=n, symmetric=form == ops.GRAD_SYMMETRIC, seed=SEED, stream_id=STREAM, row0=ROW0,
                    stream_offset=off)
    w = torch.randn(n, generator=gen, device=DEV)
    ref = ops.grad(form, X, w, mu, sigma, 0.5, 0.25)
    kw = dict(seed=SEED, row0=ROW0, scale_mu=0.5, scale_sigma=0.25, stream_offset=off)
    for split in (0, 5, ops.GRAD_SPLIT_PERIOD, -1):
        gmu, gsig = ops.grad_hybrid(form, X, w, mu, sigma, stream_id=STREAM, split=split, **kw)
        assert torch.equal(gmu, ref[0]) and torch.equal(gsig, ref[1]), split
    # the rows really are rebuilt: other counters give another result
    gmu, _ = ops.grad_hybrid(form, X, w, mu, sigma, stream_id=STREAM + 1, split=ops.GRAD_SPLIT_PERIOD, **kw)
    assert not torch.equal(gmu, ref[0])


def test_hybrid_gradient_rejects_an_unknown_split():
    X = torch.zeros(8192, 1024, device=DEV)
    w, mu, sigma = torch.zeros(8192, device=DEV), torch.zeros(1024, device=DEV), torch.ones(1024, device=DEV)
    with pytest.raises(ValueError):
        ops.grad_hybrid(ops.GRAD_SYMMETRIC, X, w, mu, sigma, seed=0, stream_id=0, row0=0, scale_mu=1.0, scale_sigma=1.0, split=17)


# ---------------------------------------------------------------------------------------------- whole searchers
def _make(kind: str):
    prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=2000, device=DEV, seed=5)
    if kind == "pgpe":
        return PGPE(prob, popsize=20000, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    return SNES(prob, popsize=20000, stdev_init=2.0)


def _reading(searcher):
    """The reference run: after the first (sampling-only) step, every gradient pass reads the stored population."""
    searcher.step()
    pop = searcher._population
    pop.gradient_samples = lambda mu, sigma: pop._data
    return searcher


def _hybrid_calls(monkeypatch) -> list:
    calls = []
    real = ops.grad_hybrid

    def counted(*args, **kwargs):
        calls.append(kwargs.get("split", -1))
        return real(*args, **kwargs)

    monkeypatch.setattr(ops, "grad_hybrid", counted)
    return calls


def _modify(searcher, how: str):
    pop = searcher._population
    if how == "add_":
        pop.access_values(keep_evals=True)[:64].add_(0.25)
    else:
        f = pop.evals[:, 0].clone()
        X = pop.values.clone()
        X[5:9] *= 1.5
        pop.set_values(X)
        pop.set_evals(f)


def _trajectory(searcher, gens: int, modify_at=(), how: str = "add_") -> list:
    out = []
    for gen in range(gens):
        if gen in modify_at:
            _modify(searcher, how)
        searcher.step()
        out.append((searcher.status["center"].clone(), searcher.status["stdev"].clone()))
    return out


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
@pytest.mark.parametrize("kind", ["pgpe", "snes"])
def test_searcher_with_rebuilt_rows_matches_the_reading_run(kind, graph, monkeypatch):
    calls = _hybrid_calls(monkeypatch)
    ref = _trajectory(_reading(_make(kind)), 5)
    assert calls == []
    s = _make(kind)
    if graph:
        s.enable_cuda_graph()
    s.step()
    got = _trajectory(s, 5)
    assert len(calls) > 0
    if graph:
        assert s._graph is not None
    for gen, ((c0, s0), (c1, s1)) in enumerate(zip(ref, got)):
        assert torch.equal(c0, c1) and torch.equal(s0, s1), gen


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
@pytest.mark.parametrize("how", ["add_", "set_values"])
def test_population_modified_in_place_is_read_not_rebuilt(how, graph):
    # modified before generations 2 and 5: in graph mode these fall between replays (capture at 0, 3)
    modify_at = (2, 5)
    ref = _trajectory(_reading(_make("pgpe")), 7, modify_at, how)
    s = _make("pgpe")
    if graph:
        s.enable_cuda_graph()
    s.step()
    got = _trajectory(s, 7, modify_at, how)
    for gen, ((c0, s0), (c1, s1)) in enumerate(zip(ref, got)):
        assert torch.equal(c0, c1) and torch.equal(s0, s1), gen
    if graph:
        assert s._graph is not None


def test_gradient_samples_record_is_dropped_by_in_place_writes():
    s = _make("pgpe")
    s.step()
    pop, dist = s._population, s._distribution
    assert not isinstance(pop.gradient_samples(dist.mu, dist.sigma), torch.Tensor)
    assert isinstance(pop.gradient_samples(dist.mu.clone(), dist.sigma), torch.Tensor)  # another tensor than the sampler read
    pop.access_values(keep_evals=True)[0, 0] += 1.0
    assert pop.gradient_samples(dist.mu, dist.sigma) is pop.access_values(keep_evals=True)
    assert isinstance(pop[0:10].gradient_samples(dist.mu, dist.sigma), torch.Tensor)  # slices carry no record
