"""Full-covariance CMA-ES on the fused path (`CMAES._step_fused`, CUDA float32), kernel by kernel and generation by generation,
against the float64 oracle (`oracle.es_oracle`: `cmaes_recombine`, `cmaes_vector_step`, `cmaes_covariance_coefficients`,
`cmaes_active_weights`, `cmaes_covariance_update`, `cmaes_decomposition_due`; pinned to the reference's own runs by
tests/test_oracle_golden.py).

Tolerance, per element:  |x - x64| <= C_ROUND * 2^-24 * K_eff * mag + aerr, where mag is the same expression evaluated on magnitudes
(|m| + sigma |Z| |A|^T for the population, sum_i |w_i| |y_i| for the recombination, ...) and K_eff the length of the longest
sum that feeds the element.  The searcher-level test also proves on its own data that the bound is tight: seven mutated references
(h_sig from steps + 1, weighted_pc dropped, the (1 - h^2) term dropped from c1a, rank-mu with the nominal weights, m moved with the
new sigma, the decomposition one generation late, an ascending rank for "max") must each fall outside it in at least one case.
"""

import math

import numpy as np
import pytest
import torch

from oracle import es_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import Problem, ops
    from evotorch_b200.algorithms import CMAES
    from evotorch_b200.objectives import sphere

DEV = "cuda"
EPS32 = 2.0**-24
# C_ROUND, calibrated once on an H100 80GB HBM3 (400 W): the largest |x - x64| / bound measured over this file was 0.50 (vector
# update: m, p_sigma, p_c; k 0.27, sigma 0.15), 0.43 (row weights), and in the generations 0.44 (X), 0.43 (m), 0.32 (C), 0.30 (p_c),
# 0.27 (p_sigma), 0.16 (A), 0.14 (sigma).  Every mutated reference still falls outside the bound in at least one case
C_ROUND = 4.0
_WORST = {}


def C(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def _ratio(got, ref, bound):
    """max |got - ref| / bound over the elements (inf where a value is not finite)."""
    got, ref, bound = (np.asarray(v, np.float64) for v in (got, ref, bound))
    err = np.abs(got - ref)
    err = np.where(np.isfinite(err), err, np.inf)
    return float(np.max(err / bound)) if err.size else 0.0


def _check(name, got, ref, bound):
    r = _ratio(got, ref, bound)
    _WORST[name] = max(_WORST.get(name, 0.0), r)
    assert r <= 1.0, f"{name}: error / bound = {r:.3g}"


def _consts(st):
    return (st.c_m, st.c_sigma, st.damp_sigma, st.c_c, st.c_1, st.c_mu, st.variance_discount_sigma, st.variance_discount_c,
            float(st.unbiased_expectation), float(np.sum(st.weights, dtype=np.float32)))


def _default_popsize(d):
    return 4 + int(np.floor(3 * np.log(d)))


# ------------------------------------------------------------------------------------------------ evok_cmaes_vector_update
@pytest.mark.parametrize("D", [1, 2, 31, 32, 33, 1023, 1024, 1025, 2049, 5000])
@pytest.mark.parametrize("csa_squared", [0, 1])
@pytest.mark.parametrize("h_target", [1.0, 0.0])
@pytest.mark.parametrize("counter", ["host", "device"])
def test_vector_update_matches_the_oracle_vector_step(D, csa_squared, h_target, counter):
    """One CTA of 1024 threads, one to five elements per thread: m, p_sigma, p_c and sigma within the bound of the oracle's vector
    step from a random state, h_sig exactly, k_out = (c_mu, 1 - c1a - c_mu sum(w), c1a c_1 / (c1a + 1e-23)).  The state is scaled
    so that ||p_sigma'||^2 lands 30 % below or above the h_sig threshold; the step count comes from the host or from the device
    counter, which must come back incremented."""
    rng = np.random.default_rng(D * 4 + csa_squared * 2 + int(h_target))
    n = max(_default_popsize(D), 6)
    st = O.CMAESState(D, n, 0.7, rng.uniform(-2, 2, D), csa_squared=bool(csa_squared))
    st.steps = steps = 3
    f32 = np.float32
    p_sigma0 = rng.standard_normal(D)
    local = rng.standard_normal(D)
    # scale p_sigma and local together so that lhs = ||p_sigma'||^2 / decay / D - 1 is rhs * (1 -+ 0.3)
    v = (1 - st.c_sigma) * p_sigma0 + st.variance_discount_sigma * local
    decay = 1 - (1 - st.c_sigma) ** (2 * steps + 1)
    rhs = 1 + 4.0 / (D + 1)
    target = (rhs * (0.7 if h_target == 1.0 else 1.3) + 1) * D * decay
    s = math.sqrt(target / float(v @ v))
    st.p_sigma = (p_sigma0 * s).astype(f32)
    local = (local * s).astype(f32)
    st.p_c = (rng.standard_normal(D) * 0.2).astype(f32)
    shaped = (rng.standard_normal(D) * 0.5).astype(f32)
    st.sigma = f32(0.7)
    m0, ps0, pc0, sig0 = st.m.copy(), st.p_sigma.copy(), st.p_c.copy(), float(st.sigma)
    m, p_sigma, p_c, sigma = C(m0), C(ps0), C(pc0), C([sig0])
    k = torch.full((3,), float("nan"), device=DEV)
    h_out = torch.full((1,), float("nan"), device=DEV)
    steps_dev = torch.tensor([steps], dtype=torch.int64, device=DEV) if counter == "device" else None
    ops.cmaes_vector_update(C(local), C(shaped), m, p_sigma, p_c, sigma, _consts(st), bool(csa_squared), k,
                            steps=steps if counter == "host" else 0, steps_dev=steps_dev, h_sig_out=h_out)
    h = O.cmaes_vector_step(st, local.astype(np.float64), shaped.astype(np.float64))
    _, margin = O.cmaes_h_sig(st, float(np.linalg.norm(st.p_sigma.astype(np.float64))))
    assert h == h_target and margin > 0.1
    assert float(h_out) == h
    if steps_dev is not None:
        assert int(steps_dev) == steps + 1
    tol = C_ROUND * EPS32
    _check("vec/m", N(m), st.m, tol * (np.abs(m0) + abs(st.c_m * sig0) * np.abs(shaped)) + 1e-30)
    _check("vec/p_sigma", N(p_sigma), st.p_sigma, tol * (abs(1 - st.c_sigma) * np.abs(ps0) + st.variance_discount_sigma * np.abs(local)) + 1e-30)
    _check("vec/p_c", N(p_c), st.p_c, tol * (abs(1 - st.c_c) * np.abs(pc0) + h * st.variance_discount_c * np.abs(shaped)) + 1e-30)
    pnorm = float(np.linalg.norm(st.p_sigma.astype(np.float64)))
    mag_expo = pnorm**2 / D if csa_squared else pnorm / st.unbiased_expectation
    _check("vec/sigma", float(sigma), float(st.sigma), tol * float(st.sigma) * (4 + (st.c_sigma / st.damp_sigma) * 4 * mag_expo))
    k_ref = O.cmaes_k(st, h)
    c1a, _ = O.cmaes_covariance_coefficients(st, h)
    wsum = float(np.sum(st.weights, dtype=np.float32))
    k_mag = (abs(st.c_mu), 1 + c1a + abs(st.c_mu * wsum), 3 * abs(k_ref[2]))
    _check("vec/k", N(k), k_ref, tol * np.array(k_mag))


# ------------------------------------------------------------------------------------------------ evok_cmaes_row_weights
@pytest.mark.parametrize("n", [1, 7, 8, 9, 4097])
@pytest.mark.parametrize("D", [1, 3, 4, 37, 64, 1025])
@pytest.mark.parametrize("layout", ["contiguous", "padded", "offset"])
@pytest.mark.parametrize("active", [0, 1])
def test_row_weights_match_float64(n, D, layout, active):
    """w_pos = max(a, 0) exactly (the sign of a zero weight is not specified: it multiplies rows in a sum) and w_act = D a / ||z||^2
    for the non-positive weights with `active` (a otherwise) within the bound, on a contiguous Z (the float4 path when D % 4 == 0),
    a padded pitch (float4 when the pitch is a multiple of 4) and a one-float offset (the scalar path).  Weights: positive, +0, -0
    and negative.  Nothing is written past N."""
    g = torch.Generator(device=DEV).manual_seed(n * 131 + D)
    pitch = {"contiguous": D, "padded": (D + 3) // 4 * 4 + 4, "offset": D + 1}[layout]
    store = torch.randn(n * pitch + 1, device=DEV, generator=g)
    base = 1 if layout == "offset" else 0
    Z = store[base:base + n * pitch].view(n, pitch)[:, :D]
    a = torch.randn(n, device=DEV, generator=g)
    kind = torch.arange(n, device=DEV) % 5
    a = torch.where(kind == 1, torch.zeros_like(a), a)
    a = torch.where(kind == 2, torch.full_like(a, -0.0), a)
    a = torch.where(kind == 3, -a.abs(), a)
    w_pos = torch.full((n + 1,), float("nan"), device=DEV)
    w_act = torch.full((n + 1,), float("nan"), device=DEV)
    ops.cmaes_row_weights(a, Z, bool(active), w_pos[:n], w_act[:n])
    assert torch.isnan(w_pos[n]) and torch.isnan(w_act[n])
    assert torch.equal(w_pos[:n], torch.clamp_min(a, 0.0))
    z64 = Z.double()
    ref = torch.where(a > 0, a.double(), D * a.double() / (z64 * z64).sum(dim=1)) if active else a.double()
    pos = a > 0
    assert torch.equal(w_act[:n][pos], a[pos])
    if not active:
        assert torch.equal(w_act[:n], a)
    _check("row_weights/w_act", N(w_act[:n]), N(ref), C_ROUND * EPS32 * D * np.abs(N(ref)) + 1e-38)


# ------------------------------------------------------------------------------------------------ searcher-level generations
def _linear(x):
    return torch.sum(x, dim=-1)


def _shifted_to_maximise(x):
    return -torch.sum((x - 1.5) ** 2 * torch.arange(1, x.shape[-1] + 1, dtype=x.dtype, device=x.device), dim=-1)


def _sphere_with_nonfinite(x):
    f = torch.sum(x**2, dim=-1)
    r = torch.arange(f.shape[0], device=x.device)
    f = torch.where(r % 7 == 3, torch.full_like(f, float("nan")), f)
    f = torch.where(r % 11 == 5, torch.full_like(f, float("inf")), f)
    return torch.where(r % 13 == 8, torch.full_like(f, float("-inf")), f)


# name: (D, sense, objective, searcher options, generations (None: 2 * decompose_C_freq + 1), seed)
CASES = {
    "D1": (1, "min", "sphere", {}, None, 1),
    "D3": (3, "min", "sphere", {}, None, 1),
    "D5": (5, "min", "sphere", {}, None, 1),
    "D200_freq2": (200, "min", "sphere", {}, None, 1),
    "D500_freq4": (500, "min", "sphere", {}, None, 1),
    "D1025_freq8": (1025, "min", "sphere", {}, None, 1),
    "D129_n8193_radix": (129, "min", "sphere", {"popsize": 8193}, None, 1),
    "consts": (40, "min", "sphere", dict(active=False, csa_squared=True, c_m=0.9, c_sigma_ratio=1.5, damp_sigma_ratio=0.8, c_c_ratio=1.2,
                                         c_1_ratio=0.5, c_mu_ratio=2.0), None, 1),
    "max_shifted": (30, "max", "shifted", {}, None, 1),
    "nonfinite": (20, "min", "nonfinite", {"popsize": 40}, None, 1),
    "linear_h0": (10, "min", "linear", {"stdev_init": 1e-3}, 14, 1),
}
MUTATIONS = ("h_steps_plus_1", "no_weighted_pc", "c1a_without_h", "nominal_rank_mu_weights", "m_with_new_sigma", "decompose_late",
             "ascending_max")
_OBJECTIVES = {"linear": _linear, "shifted": _shifted_to_maximise, "nonfinite": _sphere_with_nonfinite}
_ORACLE_KEYS = ("active", "csa_squared", "c_m", "c_sigma_ratio", "damp_sigma_ratio", "c_c_ratio", "c_1_ratio", "c_mu_ratio")


def _reference(snap, Z, Y, f, sense, okw, mutation=None):
    """One generation of the oracle from the GPU's state before it, optionally with one of MUTATIONS."""
    D, n = Z.shape[1], Z.shape[0]
    st = O.CMAESState(D, n, snap["sigma"], snap["m"], **okw)
    for key in ("C", "A", "p_sigma", "p_c"):
        setattr(st, key, snap[key].copy())
    st.sigma, st.steps = np.float32(snap["sigma"]), snap["steps"]
    aw = O.cmaes_assign_weights(st, f, "min" if mutation == "ascending_max" else sense)
    local, shaped = O.cmaes_recombine(st, Z, Y, aw)
    st.steps += mutation == "h_steps_plus_1"
    h = O.cmaes_vector_step(st, local, shaped)
    st.steps = snap["steps"]
    if mutation == "m_with_new_sigma":
        st.m = (snap["m"] + np.float32(st.c_m) * st.sigma * shaped.astype(np.float32)).astype(np.float32)
    c1a, wpc = O.cmaes_covariance_coefficients(st, h)
    if mutation == "no_weighted_pc":
        wpc = 1.0
    if mutation == "c1a_without_h":
        c1a = st.c_1 * (1 - st.c_c * (2 - st.c_c))
        wpc = (st.c_1 / (c1a + 1e-23)) ** 0.5
    w = aw.astype(np.float64) if mutation == "nominal_rank_mu_weights" else O.cmaes_active_weights(st, Z, aw)
    C_before = st.C
    O.cmaes_covariance_update(st, Y, w, c1a, wpc)
    due = O.cmaes_decomposition_due(st) if mutation != "decompose_late" else st.steps % st.decompose_C_freq == 0 and st.steps > 0
    if due:
        O.cmaes_decompose(st)
    pnorm = float(np.linalg.norm(st.p_sigma.astype(np.float64)))
    _, margin = O.cmaes_h_sig(st, pnorm)
    return dict(st=st, h=h, margin=margin, due=due, aw=aw, w_act=w, c1a=c1a, wpc=wpc, C_before=C_before, pnorm=pnorm)


def _bounds(snap, Z, Y, ref):
    """Per-element bounds of X, m, p_sigma, p_c, sigma, C and A for one generation (see the module docstring)."""
    st = ref["st"]
    n, D = Z.shape
    tol = C_ROUND * EPS32
    sig0 = float(snap["sigma"])
    Zabs = np.abs(Z)
    Ymag = Zabs @ np.abs(snap["A"].astype(np.float64)).T
    a_pos = np.maximum(ref["aw"].astype(np.float64), 0.0)
    mu = int(np.count_nonzero(a_pos))
    Sy, Sz = a_pos @ Ymag, a_pos @ Zabs
    b = {}
    # 3xTF32 drops the lo x lo products (about 2^-22 of each term): 4 more terms' worth of rounding, which weighs at small D
    b["X"] = tol * ((D + 4) * sig0 * Ymag + np.abs(snap["m"])) + 1e-30
    b["m"] = tol * (np.abs(snap["m"]) + st.c_m * sig0 * (mu + D) * Sy) + 1e-30
    b["p_sigma"] = tol * (abs(1 - st.c_sigma) * np.abs(snap["p_sigma"]) + st.variance_discount_sigma * mu * Sz) + 1e-30
    b["p_c"] = tol * (abs(1 - st.c_c) * np.abs(snap["p_c"]) + st.variance_discount_c * (mu + D) * Sy) + 1e-30
    mag_expo = ref["pnorm"] ** 2 / D if st.csa_squared else ref["pnorm"] / st.unbiased_expectation
    b["sigma"] = tol * float(st.sigma) * (4 + (st.c_sigma / st.damp_sigma) * (mu + 4) * mag_expo)
    k0, k1, k2 = st.c_mu, 1 - ref["c1a"] - st.c_mu * float(np.sum(st.weights, dtype=np.float32)), ref["c1a"] * ref["wpc"] ** 2
    pc = np.abs(st.p_c.astype(np.float64))
    S = (np.abs(ref["w_act"])[:, None] * Ymag).T @ Ymag
    b["C"] = tol * ((n + D) * k0 * S + abs(k1) * np.abs(ref["C_before"]) + 2 * (mu + D) * abs(k2) * np.outer(pc, pc) + np.abs(st.C)) + 1e-30
    dg = np.sqrt(np.abs(np.diag(st.C).astype(np.float64)))
    b["A"] = tol * (n + D) * np.outer(dg, dg) + 1e-30
    return b


def _compare(got, snap, Z, Y, ref, bounds, record=None):
    """Check (record=None) or measure (record=dict, the worst ratio of each quantity) one generation against one reference."""
    st = ref["st"]
    X64 = snap["m"].astype(np.float64) + float(snap["sigma"]) * Y
    pairs = [("X", got["X"], X64), ("m", got["m"], st.m), ("p_sigma", got["p_sigma"], st.p_sigma), ("p_c", got["p_c"], st.p_c),
             ("sigma", got["sigma"], float(st.sigma)), ("C", got["C"], st.C)]
    if ref["due"]:
        pairs.append(("A", got["A"], st.A))
    worst = 0.0
    for name, g, r in pairs:
        if record is None:
            _check(f"gen/{name}", g, r, bounds[name])
        else:
            worst = max(worst, _ratio(g, r, bounds[name]))
    if not ref["due"]:
        same = np.array_equal(got["A"], snap["A"])
        if record is None:
            assert same, "A changed on a generation without decomposition"
        elif not same:
            worst = math.inf
    return worst


_RUNS = {}


def _run_case(name):
    """Step the fused searcher through the case, check every generation against the oracle and measure every mutated reference."""
    if name in _RUNS:
        return _RUNS[name]
    D, sense, obj, kw, gens, seed = CASES[name]
    kw = dict(kw)
    stdev_init = kw.pop("stdev_init", 1.0)
    pkw = dict(vectorized=True) if obj in _OBJECTIVES else {}
    prob = Problem(sense, _OBJECTIVES.get(obj, sphere), initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=seed, **pkw)
    c = CMAES(prob, stdev_init=stdev_init, **kw)
    assert c._fused_ok()
    okw = {k: v for k, v in kw.items() if k in _ORACLE_KEYS}
    gens = gens or 2 * c.decompose_C_freq + 1
    seen = dict(h=set(), due=set(), min_margin=math.inf, popsize=c.popsize, freq=c.decompose_C_freq)
    caught = {mut: 0.0 for mut in MUTATIONS}  # the largest error / bound of each mutated reference
    for _ in range(gens):
        snap = dict(m=N(c.m).copy(), sigma=float(c.sigma), C=N(c.C).copy(), A=N(c.A).copy(), p_sigma=N(c.p_sigma).copy(),
                    p_c=N(c.p_c).copy(), steps=c._steps_count)
        c.step()
        Z = N(c._fused["zs"]).astype(np.float64)
        f = N(c.population.evals[:, 0])
        got = dict(X=N(c.population.values), m=N(c.m), p_sigma=N(c.p_sigma), p_c=N(c.p_c), sigma=float(c.sigma), C=N(c.C), A=N(c.A))
        Y = Z @ snap["A"].astype(np.float64).T
        ref = _reference(snap, Z, Y, f, sense, okw)
        bounds = _bounds(snap, Z, Y, ref)
        _compare(got, snap, Z, Y, ref, bounds)
        seen["h"].add(ref["h"])
        seen["due"].add(ref["due"])
        seen["min_margin"] = min(seen["min_margin"], ref["margin"])
        for mut in MUTATIONS:
            if caught[mut] <= 1.0:
                caught[mut] = max(caught[mut], _compare(got, snap, Z, Y, _reference(snap, Z, Y, f, sense, okw, mut), bounds, record={}))
    _RUNS[name] = (seen, caught)
    return _RUNS[name]


@pytest.mark.parametrize("case", list(CASES))
def test_fused_generations_match_the_float64_oracle(case):
    """Every generation of the fused path against the oracle run from the GPU's own state before it and fed the GPU's own z
    (`_fused["zs"]`) and fitnesses (so that close fitnesses cannot swap ranks between the two sides): the population X = m +
    sigma Z A^T (the sampling GEMM, pre-split when D % 4 != 0), m, sigma, p_sigma, p_c and C; A on decomposition generations, A
    bit-identical to before on the others.  Each case must reach what it is there for, and no generation may come within 1e-4
    (relative) of the h_sig threshold, so that the outcome does not hang on rounding."""
    seen, _ = _run_case(case)
    assert seen["min_margin"] > 1e-4, seen["min_margin"]
    if seen["freq"] > 1:
        assert seen["due"] == {True, False}, "decompositions must be both skipped and taken"
    if case == "linear_h0":
        assert seen["h"] == {0.0, 1.0}, seen["h"]
    if case == "D129_n8193_radix":
        assert seen["popsize"] > 8192
    if case.startswith("D200") or case.startswith("D500") or case.startswith("D1025"):
        assert seen["freq"] == {"D200_freq2": 2, "D500_freq4": 4, "D1025_freq8": 8}[case]


def test_every_mutated_reference_is_rejected_by_some_case():
    """The bounds above are tight enough to matter: each mutated reference falls outside them in at least one case."""
    caught = {mut: [] for mut in MUTATIONS}
    for case in CASES:
        for mut, ratio in _run_case(case)[1].items():
            if ratio > 1.0:
                caught[mut].append(case)
    print("worst error / bound:", {k: round(v, 3) for k, v in sorted(_WORST.items())})
    print("mutations caught by:", caught)
    missed = [mut for mut, cases in caught.items() if not cases]
    assert not missed, f"mutated references inside the bounds of every case: {missed}; caught: {caught}"


# ------------------------------------------------------------------------------------------------ CUDA-graph replay
def test_graph_replay_equals_eager_stepping_through_both_h_sig_values():
    """Sphere far from its optimum with a small step size (locally linear: the evolution path grows until h_sig = 0) at
    decompose_C_freq = 1: the captured generation, whose vector update reads h_sig's step count from the device counter, must give
    the same bits as eager fused stepping through generations with h_sig = 1 and h_sig = 0."""
    D = 12

    def make(graph):
        prob = Problem("min", sphere, initial_bounds=(-3, 3), solution_length=D, device=DEV, seed=7)
        c = CMAES(prob, stdev_init=1e-3, center_init=torch.full((D,), 50.0, device=DEV), limit_C_decomposition=False)
        if graph:
            c.enable_cuda_graph()
        return c

    a, b = make(False), make(True)
    hs = set()
    st = O.CMAESState(D, a.popsize, 1.0, np.zeros(D))
    for t in range(14):
        a.step(); b.step()
        st.steps = t
        h, margin = O.cmaes_h_sig(st, float(np.linalg.norm(N(a.p_sigma).astype(np.float64))))
        assert margin > 1e-4
        hs.add(h)
        for key in ("m", "C", "A", "p_sigma", "p_c", "sigma"):
            assert torch.equal(getattr(a, key), getattr(b, key)), (t, key)
    if b._graph is None:
        pytest.skip("the generation could not be captured on this build (library call not capturable)")
    assert hs == {0.0, 1.0}, hs
