"""Functional CMA-ES on the kernels: the batched GEMM family against the single calls (bits) and float64 (the K6 / K7 bound), whole
batched tells against the float64 oracle per item under a first-order bound, isolation of the items, no host synchronisation, and
convergence next to the CMAES class."""

import math

import pytest
import torch

from evotorch_b200 import Problem, ops
from evotorch_b200.algorithms import CMAES
from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_tell
from oracle.functional_cmaes_oracle import tell_bound

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
EPS = 2.0 ** -24
BM = BN = 128
BK = 32
SMS = 132
CHUNK = 4


def one_split(M, N, K):
    """True when gemm_nt's plan for this shape has one K split (the batched plan never splits)."""
    tiles = -(-M // BM) * -(-N // BN)
    total_kb = -(-K // BK)
    return tiles * 2 > SMS or total_kb < 2


def gamma(K):
    """The K6 / K7 bound factor (DESIGN, "Accuracy of K6 / K7") of a one-split product over K."""
    kbps = -(-K // BK)
    k_chunk = 2 * 3 * (BK // 8) * min(kbps, CHUNK) + -(-kbps // CHUNK)
    return 3 * 2.0 ** -20 + EPS * (k_chunk + 1 + 2)


def worst(err, bound):
    r = err / bound.clamp_min(1e-300)
    r = torch.where(torch.isfinite(err), r, torch.full_like(r, math.inf))
    return float(r.max())


def operand(items, rows, cols, g, aligned=True, shared=False):
    """fp32 (items, rows, cols) on the GPU (or (rows, cols) when shared); unaligned: a view with row pitch cols + 1 and item pitch
    rows * (cols + 1) + 1 (neither a multiple of 4 floats in general)."""
    if shared:
        return torch.randn(rows, cols, generator=g).to(DEV)
    if aligned:
        return torch.randn(items, rows, cols, generator=g).to(DEV)
    flat = torch.randn(items * (rows * (cols + 1) + 1) + 8, generator=g).to(DEV)
    return flat.as_strided((items, rows, cols), (rows * (cols + 1) + 1, cols + 1, 1), 1)


CASES = [(d, n, b) for d in (1, 3, 32, 129, 512) for n in (4, 17, 300) for b in (1, 5)]


@pytest.mark.parametrize("d,n,items", CASES)
@pytest.mark.parametrize("layout", ["aligned", "unaligned", "shared_B"])
def test_gemm_batched_sampling_product(d, n, items, layout):
    """x_b = m_b + sigma_b z_b A_b^T: per item the bits of gemm_nt with the same second output, and within the K6 bound of float64."""
    g = torch.Generator().manual_seed(d * 1000 + n * 10 + items)
    z = operand(items, n, d, g, aligned=layout != "unaligned")
    A = operand(items, d, d, g, aligned=layout != "unaligned", shared=layout == "shared_B")
    sigma = torch.rand(items, generator=g).to(DEV) + 0.5
    m = torch.randn(items, d, generator=g).to(DEV)
    y = torch.empty(items, n, d, device=DEV)
    x = torch.empty(items, n, d, device=DEV)
    ops.gemm_nt_batched(z, A, y, out2=x, alpha=sigma, bias=m)
    for b in range(items):
        Ab = A if A.ndim == 2 else A[b]
        yb, xb = torch.empty(n, d, device=DEV), torch.empty(n, d, device=DEV)
        ops.gemm_nt(z[b], Ab, yb, out2=xb, alpha=sigma[b:b + 1], bias=m[b])  # out2: the single call never splits K
        assert torch.equal(y[b], yb) and torch.equal(x[b], xb), b
    Ab = A.expand(items, d, d) if A.ndim == 2 else A
    ref = z.double() @ Ab.double().mT
    absab = z.double().abs() @ Ab.double().abs().mT
    assert worst((y.double() - ref).abs(), gamma(d) * absab) <= 1.0


@pytest.mark.parametrize("d,n,items", CASES)
def test_weighted_syrk_update_batched(d, n, items):
    """C_b <- k0 Y^T diag(w) Y + k1 C_b + k2 u u^T: the bits of weighted_syrk_update per item where its plan has one split, and
    everywhere within the K7 bound (with the epilogue's) of float64 over the fp32 operands the transposing pass builds."""
    g = torch.Generator().manual_seed(7 * d + n + items)
    Y = torch.randn(items, n, d, generator=g).to(DEV)
    w = torch.randn(items, n, generator=g).to(DEV)
    k = (torch.rand(items, 3, generator=g) + 0.1).to(DEV)
    C = torch.randn(items, d, d, generator=g).to(DEV)
    u = torch.randn(items, d, generator=g).to(DEV)
    out = ops.weighted_syrk_update_batched(Y, w, k, C, u=u)
    if one_split(d, d, n):
        for b in range(items):
            assert torch.equal(out[b], ops.weighted_syrk_update(Y[b], w[b], k[b], C[b], u=u[b])), b
    Aw = (Y * w[:, :, None]).mT.double()  # the fp32 products the pass writes, exactly
    acc, absab = Aw @ Y.double(), Aw.abs() @ Y.double().abs()
    k64 = k.double()
    uu = u.double()[:, :, None] * u.double()[:, None, :]
    ref = k64[:, 0, None, None] * acc + k64[:, 1, None, None] * C.double() + k64[:, 2, None, None] * uu
    bound = k64[:, 0, None, None] * gamma(n) * absab + EPS * (k64[:, 0, None, None] * acc.abs() + 2 * k64[:, 1, None, None] * C.double().abs()
                                                               + 3 * k64[:, 2, None, None] * uu.abs())
    assert worst((out.double() - ref).abs(), bound) <= 1.0


def test_gemm_batched_across_item_chunks():
    """70000 items (two launches of at most 65535): every item against float64 and the items around the chunk edge against gemm_nt."""
    g = torch.Generator().manual_seed(3)
    items, n, d = 70000, 4, 3
    z = torch.randn(items, n, d, generator=g).to(DEV)
    A = torch.randn(items, d, d, generator=g).to(DEV)
    sigma, m = (torch.rand(items, generator=g) + 0.5).to(DEV), torch.randn(items, d, generator=g).to(DEV)
    y, x = torch.empty_like(z), torch.empty_like(z)
    ops.gemm_nt_batched(z, A, y, out2=x, alpha=sigma, bias=m)
    ref = z.double() @ A.double().mT
    assert worst((y.double() - ref).abs(), gamma(d) * (z.double().abs() @ A.double().abs().mT)) <= 1.0
    for b in (0, 65534, 65535, 69999):
        yb, xb = torch.empty(n, d, device=DEV), torch.empty(n, d, device=DEV)
        ops.gemm_nt(z[b], A[b], yb, out2=xb, alpha=sigma[b:b + 1], bias=m[b])
        assert torch.equal(y[b], yb) and torch.equal(x[b], xb), b
    w, k, u = torch.randn(items, n, generator=g).to(DEV), torch.rand(items, 3, generator=g).to(DEV), torch.randn(items, d, generator=g).to(DEV)
    C = torch.randn(items, d, d, generator=g).to(DEV)
    out = ops.weighted_syrk_update_batched(z, w, k, C, u=u)
    for b in (0, 65535, 69999):
        assert torch.equal(out[b], ops.weighted_syrk_update(z[b], w[b], k[b], C[b], u=u[b])), b


# ------------------------------------------------------------------------------------------------ whole tells
def ellipsoid(x):
    d = x.shape[-1]
    scale = 10.0 ** (4 * torch.arange(d, device=x.device, dtype=x.dtype) / max(d - 1, 1))
    return (scale * x * x).sum(-1)


def _tell_bound(state, x, f, new):
    """Per item: (max over the state tensors of |kernel - oracle| / first-order bound), `oracle.functional_cmaes_oracle.tell_bound`."""
    return tell_bound(state, x, f, new)


@pytest.mark.parametrize("d,items", [(8, 6), (33, 4), (130, 3)])
@pytest.mark.parametrize("active,csa_squared,sense", [(True, False, "min"), (False, True, "max")])
def test_whole_tells_against_the_oracle(d, items, active, csa_squared, sense):
    """Tells from states an ellipsoid run has made ill-conditioned (cond(C) up to ~1e4), every item against the oracle under the
    first-order bound; the worst error over the bound is printed."""
    torch.manual_seed(d + items)
    sign = -1.0 if sense == "max" else 1.0
    state = cmaes(center_init=torch.randn(items, d, device=DEV) * 2, stdev_init=torch.linspace(0.5, 1.5, items, device=DEV), objective_sense=sense,
                  active=active, csa_squared=csa_squared)
    worst_ratio = 0.0
    gens = {8: 120, 33: 150, 130: 60}[d]
    for gen in range(gens):
        x = cmaes_ask(state)
        f = sign * ellipsoid(x)
        if gen % (gens // 3) == gens // 3 - 1:
            new = cmaes_tell(state, x, f)
            worst_ratio = max(worst_ratio, max(_tell_bound(state, x, f, new)))
            state = new
        else:
            state = cmaes_tell(state, x, f)
    cond = float(torch.linalg.cond(state.C.double()).max())
    print(f"d={d} items={items}: worst |err| / bound {worst_ratio:.3f}, cond(C) up to {cond:.3g}")
    assert worst_ratio <= 1.0


def test_one_item_on_the_kernels_agrees_with_the_torch_path_and_the_oracle():
    """A batch of one item: the kernels against the batched torch ops (float32, CPU) every generation, and against the oracle."""
    torch.manual_seed(0)
    d = 12
    for kw in (dict(), dict(stdev_min=0.3, stdev_max=0.8), dict(active=False, csa_squared=True)):
        sk = cmaes(center_init=torch.randn(1, d, device=DEV), stdev_init=0.5, objective_sense="min", **kw)
        for gen in range(12):
            x = cmaes_ask(sk)
            f = ellipsoid(x)
            new_k = cmaes_tell(sk, x, f)
            st = sk._replace(center=sk.center.cpu(), sigma=sk.sigma.cpu(), C=sk.C.cpu(), A=sk.A.cpu(), p_sigma=sk.p_sigma.cpu(), p_c=sk.p_c.cpu(),
                             hyperparameters=sk.hyperparameters._replace(weights=sk.hyperparameters.weights.cpu()))
            new_t = cmaes_tell(st, x.cpu(), f.cpu())
            for name in ("center", "sigma", "C", "A", "p_sigma", "p_c"):
                a, b = getattr(new_k, name).cpu().double(), getattr(new_t, name).double()
                assert torch.allclose(a, b, rtol=2e-4, atol=2e-5 * float(b.abs().max())), (kw, gen, name)
            if gen in (2, 9) and "stdev_min" not in kw:
                assert max(_tell_bound(sk, x, f, new_k)) <= 1.0
            sk = new_k


def test_isolation_of_items():
    """NaN / inf in one item's values or fitnesses leaves every other item's new state bit-identical."""
    torch.manual_seed(1)
    d, items = 10, 6
    state = cmaes(center_init=torch.randn(items, d, device=DEV), stdev_init=1.0, objective_sense="min", limit_C_decomposition=False)
    for _ in range(3):
        x = cmaes_ask(state)
        state = cmaes_tell(state, x, ellipsoid(x))
    x = cmaes_ask(state)
    f = ellipsoid(x)
    clean = cmaes_tell(state, x, f)
    xp, fp = x.clone(), f.clone()
    xp[1, 3, 2] = float("nan")
    xp[4, 0, :] = float("inf")
    fp[2, 5] = float("nan")
    fp[3, :] = float("inf")
    dirty = cmaes_tell(state, xp, fp)
    for b in (0, 5):
        for name in ("center", "sigma", "C", "A", "p_sigma", "p_c"):
            assert torch.equal(getattr(clean, name)[b], getattr(dirty, name)[b]), (b, name)


def test_ask_and_tell_never_synchronise():
    torch.manual_seed(2)
    state = cmaes(center_init=torch.randn(16, 20, device=DEV), stdev_init=1.0, objective_sense="min", limit_C_decomposition=False,
                  stdev_min=0.01, stdev_max=10.0)
    x = cmaes_ask(state)
    state = cmaes_tell(state, x, ellipsoid(x))  # warm every library handle
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            x = cmaes_ask(state)
            state = cmaes_tell(state, x, ellipsoid(x))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert state.generation == 3


def rosenbrock(x):
    return (100 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1 - x[..., :-1]) ** 2).sum(-1)


def sphere(x):
    return (x * x).sum(-1)


@pytest.mark.parametrize("name,fn,gens,spread", [("sphere", sphere, 250, 3.0), ("rosenbrock", rosenbrock, 1200, 0.5)])
def test_convergence_next_to_the_class(name, fn, gens, spread):
    """Every item of a 256-item batch (distinct centres) reaches, within `gens` generations, the fitness the CMAES class reaches on
    the same problem from some of those centres in as many generations."""
    torch.manual_seed(4)
    d, items = 10, 256
    centers = (1.0 if name == "rosenbrock" else 0.0) + spread * torch.randn(items, d, device=DEV)
    state = cmaes(center_init=centers, stdev_init=0.5, objective_sense="min")
    best = torch.full((items,), math.inf, device=DEV)
    for _ in range(gens):
        x = cmaes_ask(state)
        f = fn(x)
        best = torch.fmin(best, torch.nan_to_num(f, nan=math.inf).min(-1).values)  # (a search converged to sigma = 0 turns NaN)
        state = cmaes_tell(state, x, f)
    targets = []
    for i in range(4):
        prob = Problem("min", fn, solution_length=d, initial_bounds=(-1, 1), device=DEV, vectorized=True, seed=i)
        s = CMAES(prob, stdev_init=0.5, center_init=centers[i].clone())
        best_i = math.inf
        for _ in range(gens):
            s.step()
            best_i = min(best_i, float(s.status["pop_best_eval"]))
        targets.append(best_i)
    target = max(max(targets), 1e-9)
    reached = float((best <= target).float().mean())
    print(f"{name}: class reaches {targets}; batch worst {float(best.max()):.3g}, median {float(best.median()):.3g}, share reaching {reached:.3f}")
    if name == "sphere":
        assert float(best.max()) <= target
    else:
        # CMA-ES with the default population converges to the local minimum of the 10-D Rosenbrock function (f = 3.99, near
        # x_0 = -1) from some starts, the class as well: every item reaches the global optimum or that minimum, and most the former
        assert float(best.max()) < 3.99 + 0.01 and reached >= 0.9
