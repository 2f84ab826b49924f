"""Parity tests at the sizes and modes the hot path actually runs in (on the GPU, `-m gpu`).

  * same-seed contract: `Problem(device="cuda", rng="torch", seed=S)` + PGPE beside the reference's torch op sequence
    (`oracle/ref_cpu_path.PGPEReferencePath(device="cuda", seed=S)`, bit-identical to the live reference on CPU,
    tests/test_ref_cpu_port.py): identical populations, bit-exact ranking on tie-free generations, mu / sigma <= 1e-5
    (gaussian.py:351-367 of the reference);
  * the TMA-staged gradient kernel (the one the bench runs) against the float64 oracle at TMA-eligible shapes, both
    implementations (EVOK_GRAD_TMA = 0 / 1), and at the metric size on sampled columns (the reduction is column-separable);
  * one CMA-ES generation at BASELINE config 3 size (D = 1024, N = 4096) against `oracle.cmaes_update` (cmaes.py:519-553).
"""

import os

import numpy as np
import pytest
import torch

from oracle import es_oracle as O
from oracle.ref_cpu_path import PGPEReferencePath

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, ops
    from evotorch_b200.algorithms import CMAES, PGPE
    from evotorch_b200.objectives import rastrigin, sphere

DEV = "cuda"


def C(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def close(a, b, rtol=1e-5, atol=1e-6):
    np.testing.assert_allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=rtol, atol=atol)


# ------------------------------------------------------------------------------------------------ same seed, torch RNG
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_same_seed_torch_rng_matches_reference_path(seed):
    """North-star contract "results match the reference's own PyTorch path on the same seed".  Both sides draw from
    torch.Generator(device="cuda").manual_seed(seed) through the same strided `normal_` calls (tools/misc.py:1739-1749), so
    the populations must be IDENTICAL bit for bit, ranking indices bit-exact, mu / sigma within 1e-5 relative
    (gaussian.py:351-367).  The two sides are compared generation by generation from a COMMON state: after the 1e-5
    assertion on (mu, sigma) the reference side takes over our bits (K4 sums in another order than torch.sum, so the
    parameters agree to 1e-5 but not bitwise -- without this the next populations could not be compared bit for bit), and
    both sides rank the same fitness vector (ours; K2's summation order differs from torch.sum's in the last bits, which
    may swap a near-tie: SURVEY 7.3)."""
    n, D, gens = 2000, 300, 6
    prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=D, device=DEV, seed=seed, rng="torch")
    s = PGPE(prob, popsize=n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    ref = PGPEReferencePath(D, n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0, seed=seed, device=DEV)
    assert torch.equal(s._distribution.mu, ref.mu)  # Problem.generate_values(1) consumed the generator identically
    s.step()
    ref.step()
    tie_free = 0
    for g in range(gens):
        X, f = s.population.values, s.population.evals[:, 0]
        assert torch.equal(X, ref.X), f"generation {g}: same seed and parameters must give the same population"
        close(N(f), N(ref.f), rtol=2e-6, atol=0)  # K2 vs torch.sum
        # K3 on the reference's own fitness vector: the permutation torch.argsort returns, bit for bit
        perm = torch.empty(n, dtype=torch.int64, device=DEV)
        w = ops.rank(ref.f.contiguous(), "centered", False, perm=perm)
        assert torch.equal(perm, ref.f.argsort(descending=True, stable=True))
        if len(torch.unique(ref.f)) == n:  # tie-free: the reference's (unstable) argsort has only one answer
            tie_free += 1
            assert torch.equal(perm, ref.f.argsort(descending=True))
        expect = torch.empty_like(ref.f)
        expect[perm] = torch.arange(n, dtype=torch.float32, device=DEV) / (n - 1) - 0.5
        assert float((w - expect).abs().max()) <= 6e-8  # torch-CUDA divides by multiplying with the reciprocal: 1 ulp
        # one generation on both sides from the common (X, f)
        ref.f = f.clone()
        s.step()
        ref._update()
        mu, sg = s.status["center"].clone(), s.status["stdev"].clone()
        close(N(mu), N(ref.mu), rtol=1e-5, atol=2e-6)
        close(N(sg), N(ref.sigma), rtol=1e-5, atol=1e-7)
        close(N(s._optimizer._velocity), N(ref.velocity), rtol=1e-5, atol=2e-6)
        ref.mu, ref.sigma, ref.velocity = mu, sg, s._optimizer._velocity.clone()
        ref._sample_and_evaluate()  # the reference's sampling ops from the same parameters and the same generator stream
    assert tie_free >= 1 or n > 1000


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_same_seed_free_running_trajectories_agree(seed):
    """The same pair left free-running for 6 generations (no re-synchronisation): the first population is identical and the
    distributions stay together (a swapped near-tie moves a gradient component by O(1/N^2), so the bound is looser)."""
    n, D = 2000, 300
    prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=D, device=DEV, seed=seed, rng="torch")
    s = PGPE(prob, popsize=n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    ref = PGPEReferencePath(D, n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0, seed=seed, device=DEV)
    s.step(); ref.step()
    assert torch.equal(s.population.values, ref.X)
    for _ in range(5):
        s.step(); ref.step()
    close(N(s.status["center"]), N(ref.mu), rtol=1e-4, atol=1e-4)
    close(N(s.status["stdev"]), N(ref.sigma), rtol=1e-4, atol=1e-6)
    assert abs(float(s.status["mean_eval"]) - ref.mean_eval) < 1e-3 * abs(ref.mean_eval)


# ------------------------------------------------------------------------------------------------ K4 at TMA-eligible shapes
def _grad_oracle64(form, X, w, mu, sg, scale_mu, scale_sigma):
    w64, X64, mu64, sg64 = (a.astype(np.float64) for a in (w, X, mu, sg))
    if form == "symmetric":
        eps = X64[0::2] - mu64
        a, b = (w64[0::2] - w64[1::2]) / 2, (w64[0::2] + w64[1::2]) / 2
        g = (eps**2 - sg64**2) / sg64
    else:
        eps = X64 - mu64
        a = b = w64
        g = {"separable": (eps**2 - sg64**2) / sg64, "exp": (eps / sg64) ** 2 - 1}[form]
    ref_m = scale_mu * (a[:, None] * eps).sum(0)
    ref_s = scale_sigma * (b[:, None] * g).sum(0)
    tol_m = 3e-6 * scale_mu * (np.abs(a)[:, None] * np.abs(eps)).sum(0).max() + 1e-9
    tol_s = 3e-6 * scale_sigma * (np.abs(b)[:, None] * (np.abs(g) + 1)).sum(0).max() + 1e-9
    return ref_m, ref_s, tol_m, tol_s


@pytest.mark.parametrize("tma", ["0", "1"])
@pytest.mark.parametrize("form", ["symmetric", "separable", "exp"])
@pytest.mark.parametrize("n,D", [(8192, 1024), (20000, 2000), (16384, 10000)])
def test_grad_kernel_matches_oracle_at_tma_shapes(form, n, D, tma):
    """The bulk-copy (cp.async.bulk + mbarrier ring) gradient kernel -- the one bench.py runs -- and the LDG kernel,
    each directly against the float64 oracle (distributions.py:548-579, :708-773, :783-793)."""
    rng = np.random.default_rng(n + D)
    mu = rng.standard_normal(D).astype(np.float32)
    sg = (np.abs(rng.standard_normal(D)) * 0.5 + 0.2).astype(np.float32)
    X = (mu + sg * rng.standard_normal((n, D), dtype=np.float32)).astype(np.float32)
    w = (rng.standard_normal(n) / n).astype(np.float32)
    fid = {"separable": ops.GRAD_SEPARABLE, "symmetric": ops.GRAD_SYMMETRIC, "exp": ops.GRAD_EXP}[form]
    old = os.environ.get("EVOK_GRAD_TMA")
    os.environ["EVOK_GRAD_TMA"] = tma
    try:
        gm, gs = ops.grad(fid, C(X), C(w), C(mu), C(sg), 0.5, 2.0)
        torch.cuda.synchronize()
    finally:
        if old is None:
            os.environ.pop("EVOK_GRAD_TMA", None)
        else:
            os.environ["EVOK_GRAD_TMA"] = old
    ref_m, ref_s, tol_m, tol_s = _grad_oracle64(form, X, w, mu, sg, 0.5, 2.0)
    close(N(gm), ref_m, rtol=1e-4, atol=tol_m)
    close(N(gs), ref_s, rtol=1e-4, atol=tol_s)


def test_metric_size_gradient_matches_float64_oracle_on_sampled_columns():
    """BASELINE metric size (1 M x 10 k): K4's result on 64 sampled columns against the float64 oracle evaluated on exactly
    those columns of the stored population (the reduction is column-separable, distributions.py:763-768)."""
    free, _total = torch.cuda.mem_get_info()
    if free < 60e9:
        pytest.skip("needs 60 GB of free device memory")
    n, D = 1_000_000, 10_000
    prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=D, device=DEV, seed=11)
    s = PGPE(prob, popsize=n, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0)
    s.step()
    X, f = s.population.values, s.population.evals[:, 0]
    d = s._distribution
    w = ops.rank(f.contiguous(), "centered", False)
    g = d._compute_gradients(X, w, "centered")
    cols = np.sort(np.random.default_rng(5).choice(D, 64, replace=False))
    cols = np.concatenate([cols, [0, 1, 2, 3, D - 4, D - 3, D - 2, D - 1]])  # plus the first / last column groups
    tc = torch.as_tensor(cols, device=DEV)
    Xc = N(X[:, tc])  # 1 M x 72 floats
    ref = O.grad_symmetric(Xc, N(w), N(d.mu)[cols], N(d.sigma)[cols], "centered", "num_directions", "num_directions")
    a = (N(w)[0::2].astype(np.float64) - N(w)[1::2]) / 2
    scale = np.abs(a).sum() / (n // 2)
    close(N(g["mu"])[cols], ref["mu"], rtol=2e-4, atol=3e-6 * scale * 4)
    close(N(g["sigma"])[cols], ref["sigma"], rtol=2e-4, atol=3e-6 * scale * 16)


# ------------------------------------------------------------------------------------------------ CMA-ES at config-3 size
def test_cmaes_generation_at_config3_size_matches_oracle():
    """One CMA-ES generation at BASELINE config 3 (D = 1024, popsize = 4096, sphere) with recorded z draws: the sampling GEMM
    (Y = Z A^T with a non-trivial A), K2 / K3, the weighted recombination, the rank-mu SYRK over all 4096 rows (split-K, the
    chunked round-to-nearest accumulation) with the fused C update, and the Cholesky factor, against `oracle.cmaes_update`
    in float64 (cmaes.py:408-606): m, sigma, C, A within 2e-5."""
    D, n = 1024, 4096
    rng = np.random.default_rng(3)
    m0 = rng.uniform(-3, 3, D).astype(np.float32)
    # a non-trivial covariance to start from: C0 = B B^T / D + I with a dense B; A0 = chol(C0)
    B = rng.standard_normal((D, D))
    C0 = (B @ B.T / D + np.eye(D)).astype(np.float32)
    A0 = np.linalg.cholesky(C0.astype(np.float64)).astype(np.float32)
    Z = rng.standard_normal((n, D), dtype=np.float32)

    prob = Problem("min", sphere, initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=3)
    c = CMAES(prob, stdev_init=1.0, popsize=n, center_init=C(m0))
    c.C, c.A = C(C0), C(A0)
    zt = C(Z)
    c.sample_distribution = _recorded_sampler(c, zt)
    c.step()
    f_ours = N(c.population.evals[:, 0])

    st = O.CMAESState(D, n, 1.0, m0)
    st.C, st.A = C0.copy(), A0.copy()
    close(N(c.weights), st.weights, rtol=2e-6, atol=1e-9)
    Y, X = O.cmaes_sample(st, Z)
    close(N(c.population.values), X, rtol=2e-5, atol=2e-5)  # the sampling GEMM with its affine epilogue
    close(f_ours, O.sphere(X), rtol=2e-5)
    # both sides rank the same fitness vector: 4096 fitnesses of magnitude 1e4 are ~0.1 apart, so the 1e-6 relative difference
    # between K2 and the float64 oracle swaps a few neighbouring ranks, and ONE swapped pair moves the recombination by 1e-6
    # absolute -- the ranking itself is pinned bit-exactly elsewhere (SURVEY 7.3: feed the same f to both sides)
    aw = O.cmaes_assign_weights(st, f_ours, "min")
    O.cmaes_update(st, Z, Y, aw)

    close(N(c.m), st.m, rtol=2e-5, atol=3e-6)
    close(float(c.sigma), float(st.sigma), rtol=2e-5)
    close(N(c.p_sigma), st.p_sigma, rtol=2e-5, atol=1e-5)  # = 27.8 (variance discount) x the fp32 weighted row sum
    close(N(c.p_c), st.p_c, rtol=2e-5, atol=1e-5)
    scale = float(np.abs(st.C).max())
    assert float(np.abs(N(c.C).astype(np.float64) - st.C).max()) <= 2e-5 * scale
    assert float(np.abs(N(c.A).astype(np.float64) - st.A).max()) <= 2e-5 * float(np.abs(st.A).max())


def _recorded_sampler(c, zt):
    """sample_distribution with the z draws replaced by a recording; Y and X go through the product's own GEMM path."""
    def sample(num_samples=None):
        ys = torch.empty_like(zt)
        xs = torch.empty_like(zt)
        ops.gemm_nt(zt, c.A.contiguous(), ys, out2=xs, alpha=c.sigma.reshape(1), bias=c.m.contiguous())
        return zt, ys, xs

    return sample


# ------------------------------------------------------------------------------------------------ advisor regressions
def test_sampler_writes_the_philox_known_answer():
    """Seed 0, stream 0, direction 0, columns 0..3 is Random123's first known-answer vector (counter 0, key 0): the kernel
    must write its Box-Muller image (oracle restatement pinned by tests/test_oracle_golden.py)."""
    X = torch.empty(2, 4, device=DEV)
    ops.sample_eval(ops.OBJ_NONE, X, torch.zeros(4, device=DEV), torch.ones(4, device=DEV), n_rows=2, symmetric=True, seed=0, stream_id=0)
    x, y, z, w = 0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8

    def bm(a, b):
        u1 = a * 2.0**-32 + 2.0**-33
        th = 2 * np.pi * (b * 2.0**-32 + 2.0**-33)
        r = np.sqrt(-2 * np.log(u1))
        return r * np.cos(th), r * np.sin(th)

    expect = np.array([*bm(x, y), *bm(z, w)])
    close(N(X[0]), expect, rtol=0, atol=2e-5)
    close(N(X[1]), -expect, rtol=0, atol=2e-5)


def test_before_eval_hook_sees_and_edits_the_fresh_population():
    """core.py:2559 of the reference: the hook runs inside evaluate(), AFTER distribution.sample -- it must see the new
    samples and its edits must be what gets evaluated (with hooks registered the sample and evaluate kernels are not fused)."""
    D, n = 64, 256
    prob = Problem("min", sphere, initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=4)
    seen = []

    def hook(batch):
        v = batch.access_values(keep_evals=True)
        seen.append(v.clone())
        v.clamp_(-0.5, 0.5)

    prob.before_eval_hook.append(hook)
    s = PGPE(prob, popsize=n, center_learning_rate=0.3, stdev_learning_rate=0.1, stdev_init=1.0).enable_cuda_graph()
    for g in range(4):
        s.step()
        X, f = s.population.values, s.population.evals[:, 0]
        assert float(X.abs().max()) <= 0.5  # the edit survived
        close(N(f), O.sphere(N(X)), rtol=1e-5)  # and is what was evaluated
        assert len(seen) == g + 1 and float(seen[-1].abs().max()) > 0.5  # the hook saw the fresh, unclamped samples
        if g > 0:
            assert not torch.equal(seen[-1], seen[-2])
    assert s._graph is None  # a Python hook cannot be replayed: the searcher stayed on the eager path


def test_captured_graph_owns_its_workspaces():
    """A CUDA graph bakes raw workspace pointers in.  A later, larger workspace request (here: ranking a bigger vector and a
    second searcher) must not invalidate the memory a captured graph still writes to: the replayed trajectory stays
    bit-identical to eager stepping."""
    def make():
        prob = Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=512, device=DEV, seed=9)
        return PGPE(prob, popsize=20_000, center_learning_rate=0.4, stdev_learning_rate=0.1, stdev_init=1.0)

    eager, graph = make(), make().enable_cuda_graph()
    for _ in range(3):
        eager.step(); graph.step()
    assert graph._graph is not None
    # bigger requests on every shared workspace tag, then garbage that would land in recycled memory
    big = torch.randn(3_000_000, device=DEV)
    ops.rank(big, "centered", False)
    other = PGPE(Problem("min", rastrigin, initial_bounds=(-5.12, 5.12), solution_length=4096, device=DEV, seed=1), popsize=60_000,
                 center_learning_rate=0.4, stdev_learning_rate=0.1, stdev_init=1.0)
    other.run(3)
    del big
    torch.cuda.empty_cache()
    junk = [torch.full((1 << 22,), float("nan"), device=DEV) for _ in range(8)]
    for _ in range(3):
        eager.step(); graph.step(); other.step()
        for j in junk:
            j.fill_(float("nan"))
    assert torch.equal(eager.status["center"], graph.status["center"]) and torch.equal(eager.status["stdev"], graph.status["stdev"])


# ------------------------------------------------------------------------------------------------ sharded ranking
@pytest.mark.parametrize("method", ["centered", "linear", "nes"])
@pytest.mark.parametrize("hib", [False, True])
@pytest.mark.parametrize("counts", [[5000, 3000, 4096, 2], [2048, 2048], [7, 0, 12001, 30, 1, 600, 2, 2050], [20000]])
def test_sharded_ranking_is_bit_identical_to_the_global_sort(method, hib, counts):
    """evok_rank_sharded with `world` simulated ranks on one GPU (one stream and one set of exchange buffers per rank, all
    resident on this device): every rank sorts only its shard, the sorted keys are exchanged, and the utilities of the local
    rows must equal -- bit for bit -- the slice of the global ranking (K3 on the concatenated vector; stable ties by global
    index, NaN largest, -0 == +0)."""
    import ctypes

    from evotorch_b200 import _native as nat

    lib = nat.lib()
    R, n = len(counts), sum(counts)
    g = torch.Generator(device=DEV).manual_seed(n + R)
    f = torch.randn(n, device=DEV, generator=g)
    f = torch.round(f * 50) / 50  # massive ties, within and across shards
    f[::97] = float("nan")
    f[5::101] = -0.0
    f[6::101] = 0.0
    offs = [0]
    for c in counts:
        offs.append(offs[-1] + c)
    want = ops.rank(f.contiguous(), method, hib)
    keys = [torch.zeros(n, dtype=torch.int32, device=DEV) for _ in range(R)]
    fsum = [torch.zeros(R, dtype=torch.float64, device=DEV) for _ in range(R)]
    flags = [torch.zeros(R, dtype=torch.int64, device=DEV) for _ in range(R)]
    epoch = [torch.zeros(1, dtype=torch.int64, device=DEV) for _ in range(R)]
    done = [torch.zeros(4, dtype=torch.int32, device=DEV) for _ in range(R)]
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    w = [torch.full((max(c, 1),), 7.0, device=DEV) for c in counts]
    mean = [torch.zeros(1, device=DEV) for _ in range(R)]
    ws = [torch.empty(lib.evok_rank_workspace_bytes(max(c, 1)), dtype=torch.uint8, device=DEV) for c in counts]
    streams = [torch.cuda.Stream() for _ in range(R)]
    tab = lambda ts: (ctypes.c_void_p * R)(*[t.data_ptr() for t in ts])
    c_offs = (ctypes.c_int64 * (R + 1))(*offs)
    torch.cuda.synchronize()
    for rounds in range(2):  # twice: the epochs / counters must come back ready for the next generation
        for r in range(R):
            fl = f[offs[r]:offs[r + 1]].contiguous() if counts[r] else torch.zeros(1, device=DEV)
            with torch.cuda.stream(streams[r]):
                rc = lib.evok_rank_sharded(ops.RANK_IDS[method], fl.data_ptr(), n, int(hib), R, r, c_offs, tab(keys), tab(fsum), tab(flags),
                                           epoch[r].data_ptr(), done[r].data_ptr(), err.data_ptr(), int(5e9), w[r].data_ptr(), mean[r].data_ptr(),
                                           ws[r].data_ptr(), ws[r].numel(), streams[r].cuda_stream)
            assert rc == 0
        torch.cuda.synchronize()
        assert int(err.item()) == 0
        for r in range(R):
            assert torch.equal(w[r][:counts[r]].view(torch.int32), want[offs[r]:offs[r + 1]].view(torch.int32)), (r, rounds)
            assert int(epoch[r].item()) == rounds + 1 and int(done[r].abs().sum().item()) == 0
    finite = f[torch.isfinite(f)]
    # the global mean is the same number on every rank (NaN here, because the vector holds NaNs; check the mechanism on a clean one)
    f2 = torch.randn(n, device=DEV, generator=g) + 3.0
    for r in range(R):
        fl = f2[offs[r]:offs[r + 1]].contiguous() if counts[r] else torch.zeros(1, device=DEV)
        with torch.cuda.stream(streams[r]):
            lib.evok_rank_sharded(ops.RANK_IDS[method], fl.data_ptr(), n, int(hib), R, r, c_offs, tab(keys), tab(fsum), tab(flags), epoch[r].data_ptr(),
                                  done[r].data_ptr(), err.data_ptr(), int(5e9), w[r].data_ptr(), mean[r].data_ptr(), ws[r].data_ptr(), ws[r].numel(),
                                  streams[r].cuda_stream)
    torch.cuda.synchronize()
    assert all(torch.equal(mean[0], m) for m in mean)
    close(float(mean[0]), float(f2.double().mean()), rtol=1e-6)
    del finite


# ------------------------------------------------------------------------------------------------ CMA-ES fused generation
def _cma(seed=5, D=96, n=384, graph=False, fused=True, **kw):
    prob = Problem("min", sphere, initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=seed)
    c = CMAES(prob, stdev_init=1.0, popsize=n, **kw)
    if not fused:
        c._fused_ok = lambda: False  # the op-by-op mirror of the reference's _step
    if graph:
        c.enable_cuda_graph()
    return c


@pytest.mark.parametrize("kw", [{}, {"active": False}, {"csa_squared": True}, {"limit_C_decomposition": False}])
def test_cmaes_fused_generation_equals_the_op_by_op_path(kw):
    """The fused generation (rank-to-weights, row weights, one vector-update kernel, covariance update in the SYRK epilogue)
    against the op-by-op mirror of the reference's `_step` (cmaes.py:567-606), same Philox draws: m, sigma, C, A, paths."""
    a, b = _cma(fused=True, **kw), _cma(fused=False, **kw)
    for g in range(6):
        a.step(); b.step()
        close(N(a.m), N(b.m), rtol=2e-5, atol=2e-6)
        close(float(a.sigma), float(b.sigma), rtol=2e-5)
        close(N(a.p_sigma), N(b.p_sigma), rtol=2e-5, atol=2e-5)
        close(N(a.p_c), N(b.p_c), rtol=2e-5, atol=2e-5)
        close(N(a.C), N(b.C), rtol=2e-5, atol=2e-6)
        close(N(a.A), N(b.A), rtol=5e-5, atol=5e-6)


def test_cmaes_cuda_graph_replay_equals_eager_stepping():
    """`enable_cuda_graph()`: the whole generation (cuSOLVER Cholesky included) replayed from one graph launch must give the
    same bits as eager fused stepping (device-side Philox generation counter and step counter)."""
    a, b = _cma(D=128, n=512, limit_C_decomposition=False), _cma(D=128, n=512, limit_C_decomposition=False, graph=True)
    for g in range(8):
        a.step(); b.step()
    if b._graph is None:
        pytest.skip("the generation could not be captured on this build (library call not capturable)")
    assert torch.equal(a.m, b.m) and torch.equal(a.C, b.C) and torch.equal(a.A, b.A) and torch.equal(a.p_sigma, b.p_sigma)
    assert float(a.sigma) == float(b.sigma) and a.status["mean_eval"] == b.status["mean_eval"]
    assert b.status["iter"] == 8


def test_rank_table_and_affine_syrk_kernels():
    """evok_rank_table == weights[rank] by argsort / scatter / gather (cmaes.py:445-451) bit for bit; evok_gemm_nt_affine ==
    k0 Y^T diag(w) Y + k1 C + k2 u u^T in float64 (direct epilogue and split-K reduction, in place).  The ranking runs on both
    sides of the counting / radix switch (8192 / 8193) with +-0, NaN and +-inf keys in both senses; the SYRK also at the (d, n)
    shapes CMA-ES runs (default popsizes, 8193 rows), in place, into a separate `out` and without the rank-1 vector."""
    g = torch.Generator(device=DEV).manual_seed(3)
    for n in (12, 4096, 8192, 8193, 20000):
        for special in (False, True):
            f = torch.round(torch.randn(n, device=DEV, generator=g) * 100) / 100
            if special:  # stable ties between +0 and -0, NaN ranked as the largest value, both infinities
                vals = torch.tensor([0.0, -0.0, float("nan"), float("inf"), float("-inf")], device=DEV)
                pick = torch.randint(0, 6, (n,), device=DEV, generator=g)
                f = torch.where(pick < 5, vals[pick.clamp_max(4)], f)
            table = torch.randn(n, device=DEV, generator=g)
            for desc in (False, True):
                idx = torch.argsort(f, descending=desc, stable=True)
                ranks = torch.empty_like(idx)
                ranks[idx] = torch.arange(n, device=DEV)
                assert torch.equal(ops.rank_table(f, desc, table), table[ranks]), (n, special, desc)
    for n, d in ((12, 6), (4096, 1024), (300, 130), (5000, 256), (4, 1), (7, 3), (14, 33), (19, 200), (24, 1025), (8193, 129), (1000, 200)):
        Y = torch.randn(n, d, device=DEV, generator=g)
        w = torch.randn(n, device=DEV, generator=g) / n
        Cm = torch.randn(d, d, device=DEV, generator=g)
        u = torch.randn(d, device=DEV, generator=g)
        k = torch.tensor([0.7, 0.9, 0.05], device=DEV)
        S = 0.7 * (Y.double().T * w.double()) @ Y.double() + 0.9 * Cm.double()
        for uu in (u, None):
            ref = S + 0.05 * torch.outer(u.double(), u.double()) if uu is not None else S
            out = ops.weighted_syrk_update(Y, w, k, Cm, u=uu)
            scale = float(ref.abs().max())
            assert float((out.double() - ref).abs().max()) / scale < 3e-6, (n, d, uu is None)
            sep = torch.full_like(Cm, float("nan"))
            assert ops.weighted_syrk_update(Y, w, k, Cm, u=uu, out=sep) is sep and torch.equal(sep, out)
            C2 = Cm.clone()
            ops.weighted_syrk_update(Y, w, k, C2, u=uu, out=C2)  # in place
            assert torch.equal(C2, out)


# ------------------------------------------------------------------------------------------------ batched functional kernels
@pytest.mark.parametrize("shape", [(5, 40, 12), (3, 1000, 100), (2, 20000, 64), (1, 30, 7), (2, 524290, 8)])
def test_batched_stage_kernels_equal_the_per_item_kernels(shape):
    """SURVEY 8(f2): every batched stage (grid y / z = batch item) computes exactly what its single-search entry point computes per
    item: K1 bit-identical, K3 bit-identical, K4 / K5 to fp32 summation order."""
    B, n, d = shape
    g = torch.Generator(device=DEV).manual_seed(B * n + d)
    mu = torch.randn(B, d, device=DEV, generator=g)
    sg = torch.rand(B, d, device=DEV, generator=g) + 0.5
    for sym in (True, False):
        X = torch.empty(B, n, d, device=DEV)
        ops.sample_batched(X, mu, sg, symmetric=sym, seed=77, stream_id0=3)
        for b in range(B):
            ref = torch.empty(n, d, device=DEV)
            ops.sample_eval(ops.OBJ_NONE, ref, mu[b].contiguous(), sg[b].contiguous(), n_rows=n, symmetric=sym, seed=77, stream_id=3 + b)
            assert torch.equal(X[b], ref)
        Xs = torch.empty(B, n, d, device=DEV)
        ops.sample_batched(Xs, mu[0].contiguous(), sg[0].contiguous(), symmetric=sym, seed=77)  # shared centre / stdev
        ref = torch.empty(n, d, device=DEV)
        ops.sample_eval(ops.OBJ_NONE, ref, mu[0].contiguous(), sg[0].contiguous(), n_rows=n, symmetric=sym, seed=77, stream_id=B - 1)
        assert torch.equal(Xs[B - 1], ref)
    f = torch.round(torch.randn(B, n, device=DEV, generator=g) * 20) / 20
    for method in METHODS_ALL:
        for hib in (False, True):
            w = ops.rank_batched(f, method, hib)
            for b in range(B):
                assert torch.equal(w[b], ops.rank(f[b].contiguous(), method, hib)), (method, hib, b)
    wm = ops.rank_batched(f, "raw", True)
    mask = ops.elite_mask_batched(wm, max(1, n // 4))
    for b in range(B):
        assert torch.equal(mask[b], ops.elite_mask(wm[b].contiguous(), max(1, n // 4)))
    w = ops.rank_batched(f, "nes", False)
    w2 = w.clone()
    ops.weights_adjust_batched_(w2, 1)
    for b in range(B):
        assert torch.equal(w2[b], ops.weights_adjust_(w[b].clone(), 1))
    for form in (ops.GRAD_SYMMETRIC, ops.GRAD_SEPARABLE, ops.GRAD_EXP, ops.GRAD_MOMENTS):
        gm, gs = ops.grad_batched(form, X, w, mu, sg, 0.5, 2.0)
        for b in range(B):
            rm, rs = ops.grad(form, X[b], w[b].contiguous(), mu[b].contiguous(), sg[b].contiguous(), 0.5, 2.0)
            close(N(gm[b]), N(rm), rtol=1e-4, atol=1e-6 * float(rm.abs().max()) + 1e-9)
            close(N(gs[b]), N(rs), rtol=1e-4, atol=1e-6 * float(rs.abs().max()) + 1e-9)
    gm, gs = ops.grad_batched(ops.GRAD_SEPARABLE, X, w, mu[0].contiguous(), sg[0].contiguous(), 1.0, 1.0)  # shared centre / stdev
    rm, rs = ops.grad(ops.GRAD_SEPARABLE, X[B - 1], w[B - 1].contiguous(), mu[0].contiguous(), sg[0].contiguous(), 1.0, 1.0)
    close(N(gm[B - 1]), N(rm), rtol=1e-4, atol=1e-6 * float(rm.abs().max()) + 1e-9)
    # K5
    grad = torch.randn(B, d, device=DEV, generator=g)
    vel, cen = torch.randn(B, d, device=DEV, generator=g) * 0.1, mu.clone()
    v2, c2 = vel.clone(), cen.clone()
    lrs, moms, caps = [0.1 + 0.01 * b for b in range(B)], [0.9 - 0.05 * b for b in range(B)], [0.15 + 0.02 * b for b in range(B)]
    ops.clipup_batched_(grad, vel, cen, lrs, moms, caps)
    for b in range(B):
        vb, cb = v2[b].clone(), c2[b].clone()
        ops.clipup_step(grad[b].contiguous(), vb, lrs[b], moms[b], caps[b], mu=cb)
        assert torch.equal(vb, vel[b]) and torch.equal(cb, cen[b])
    s1, lb, ub, mc = sg.clone(), torch.full_like(sg, 0.3), torch.full_like(sg, 1.2), torch.full_like(sg, 0.2)
    s2 = s1.clone()
    ops.sigma_update_batched_(s1, grad, lrs, False, lb=lb, ub=ub, max_change=mc)
    for b in range(B):
        sb = s2[b].clone()
        ops.sigma_update_(sb, grad[b].contiguous(), lrs[b], False, lb=lb[b], ub=ub[b], max_change=mc[b])
        assert torch.equal(sb, s1[b])


METHODS_ALL = ("centered", "linear", "nes", "normalized", "raw")


def test_functional_batched_tell_equals_the_per_item_loop(monkeypatch):
    from evotorch_b200.algorithms.functional import cem, cem_tell, pgpe, pgpe_ask, pgpe_tell

    torch.manual_seed(1)
    center = torch.randn(6, 50, device=DEV)
    st = pgpe(center_init=center, center_learning_rate=torch.linspace(0.05, 0.2, 6), stdev_learning_rate=torch.linspace(0.05, 0.15, 6),
              objective_sense="min", stdev_init=1.0, ranking_method="nes")
    x = pgpe_ask(st, popsize=200)
    ev = torch.sum(x * x, dim=-1)
    a = pgpe_tell(st, x, ev)
    monkeypatch.setenv("EVOTORCH_B200_FUNCTIONAL_LOOP", "1")
    b = pgpe_tell(st, x, ev)
    close(N(a.optimizer_state.center), N(b.optimizer_state.center), rtol=1e-5, atol=1e-6)
    close(N(a.stdev), N(b.stdev), rtol=1e-5, atol=1e-7)
    monkeypatch.setenv("EVOTORCH_B200_FUNCTIONAL_LOOP", "0")
    cs = cem(center_init=center, parenthood_ratio=0.25, objective_sense="min", stdev_init=1.0, stdev_max_change=0.3)
    a = cem_tell(cs, x, ev)
    monkeypatch.setenv("EVOTORCH_B200_FUNCTIONAL_LOOP", "1")
    b = cem_tell(cs, x, ev)
    close(N(a.center), N(b.center), rtol=1e-5, atol=1e-6)
    close(N(a.stdev), N(b.stdev), rtol=1e-5, atol=1e-7)


# ------------------------------------------------------------------------------------------------ Cholesky kernel
@pytest.mark.parametrize("n", [1, 5, 32, 33, 64, 65, 100, 128, 130, 257, 1000, 1024, 2048])
def test_tile_dataflow_cholesky_matches_float64(n):
    """evok_cholesky (cmaes.py:555-565 `decompose_C`) against numpy's float64 factorisation: L lower-triangular with zeros above
    the diagonal, L L^T = A to fp32 accuracy; only the lower triangle of the input is read."""
    g = torch.Generator(device=DEV).manual_seed(n)
    B = torch.randn(n, n, device=DEV, generator=g)
    A = (B @ B.T / n + torch.eye(n, device=DEV) * (0.5 + torch.rand(n, device=DEV, generator=g))).contiguous()
    ref = np.linalg.cholesky(N(A).astype(np.float64))
    L = ops.cholesky(A)
    assert float(torch.triu(L, 1).abs().max()) == 0.0 if n > 1 else True
    scale = float(np.abs(ref).max())
    assert float(np.abs(N(L).astype(np.float64) - ref).max()) <= 2e-5 * scale
    rec = (L.double() @ L.double().T - A.double()).abs().max() / A.double().abs().max()
    assert float(rec) < 5e-6
    # garbage above the diagonal of the input must not matter; a padded (strided) input / output works too
    junk = A + torch.triu(torch.full_like(A, 7.0), 1)
    assert torch.equal(ops.cholesky(junk), L)
    wide = torch.zeros(n, n + 4, device=DEV)
    wide[:, :n] = A
    out = torch.full((n, n + 8), 3.0, device=DEV)
    ops.cholesky(wide[:, :n], out=out[:, :n])
    assert torch.equal(out[:, :n], L) and float(out[:, n:].min()) == 3.0
    # run it twice back to back (flags are reset by every call) and against the library
    assert torch.equal(ops.cholesky(A), L)
    lib = torch.linalg.cholesky(A)
    assert float((L - lib).abs().max()) <= 2e-5 * scale


def test_cholesky_of_an_indefinite_matrix_gives_nans_not_a_hang():
    A = torch.eye(200, device=DEV)
    A[150, 150] = -1.0
    L = ops.cholesky(A)
    torch.cuda.synchronize()
    assert bool(torch.isnan(L).any())


# ------------------------------------------------------------------------------------------------ shared-minibatch policy forward
@pytest.mark.parametrize("dims,acts,n,B", [((376, 256, 17), ("tanh", "none"), 300, 70), ((6, 16, 3), ("relu", "none"), 1000, 256),
                                           ((33, 40, 24, 5), ("tanh", "sigmoid", "none"), 97, 31), ((8, 512, 2), ("none", "tanh"), 64, 300)])
def test_shared_minibatch_forward_matches_float64_and_vmap(dims, acts, n, B):
    """`Policy.forward_shared` on CUDA (first layer = tensor-core product of the stacked weight rows, gathered from odd-length,
    4-byte-aligned parameter rows) against a float64 evaluation of the same networks and against vmap(functional_call)
    (what `SupervisedNE` costs the reference per solution: supervisedne.py:250, neproblem.py:342-363)."""
    from evotorch_b200.neuroevolution import Policy

    layers = []
    for l in range(len(acts)):
        layers.append(torch.nn.Linear(dims[l], dims[l + 1]))
        if acts[l] != "none":
            layers.append({"tanh": torch.nn.Tanh, "relu": torch.nn.ReLU, "sigmoid": torch.nn.Sigmoid}[acts[l]]())
    pol = Policy(torch.nn.Sequential(*layers).to(DEV))
    g = torch.Generator(device=DEV).manual_seed(n + B)
    P = torch.randn(n, pol.parameter_length, device=DEV, generator=g) * 0.3
    x = torch.randn(B, dims[0], device=DEV, generator=g)
    y = pol.forward_shared(P, x)
    assert y.shape == (n, B, dims[-1])
    # float64 reference
    h = x.double().unsqueeze(0).expand(n, B, dims[0])
    off = 0
    for l in range(len(acts)):
        W = P[:, off:off + dims[l] * dims[l + 1]].double().view(n, dims[l + 1], dims[l])
        off += dims[l] * dims[l + 1]
        b = P[:, off:off + dims[l + 1]].double()
        off += dims[l + 1]
        h = torch.einsum("nbi,noi->nbo", h, W) + b[:, None, :]
        h = {"tanh": torch.tanh, "relu": torch.relu, "sigmoid": torch.sigmoid, "none": lambda t: t}[acts[l]](h)
    scale = float(h.abs().max())
    assert float((y.double() - h).abs().max()) <= 2e-5 * max(scale, 1.0)
    ref = torch.vmap(pol._call_one, in_dims=(0, None))(P, x)
    assert float((y - ref).abs().max()) <= 2e-5 * max(scale, 1.0)
    # a padded (strided) population and a strided batch: the same networks at other alignments.  The K axis of a tile is cut at the
    # 16-byte boundaries of ITS rows, so the summation order -- not the result beyond rounding -- depends on the alignment; junk in
    # the padding (NaN) must not leak into any row
    for pad in (1, 2, 3, 4):
        wideP = torch.full((n, pol.parameter_length + pad), float("nan"), device=DEV)
        wideP[:, :pol.parameter_length] = P
        widex = torch.full((B, dims[0] + 5), float("nan"), device=DEV)
        widex[:, :dims[0]] = x
        y2 = pol.forward_shared(wideP[:, :pol.parameter_length], widex[:, :dims[0]])
        assert float((y2 - y).abs().max()) <= 2e-5 * max(scale, 1.0)
    # the same call twice gives the same bits
    assert torch.equal(pol.forward_shared(P, x), y)
