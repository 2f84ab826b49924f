"""The batched stages of the functional ask / tell API (`evok_*_batched`, include/evok.h) and the per-item K5 kernels it uses, stage by
stage and tell by tell, against the float64 oracle (oracle/functional_oracle.py, itself checked against the reference and the float64
torch path in tests/test_functional_oracle.py), at batch sizes that reach the item chunking: 256 items per launch for the K5 stages,
65535 (the grid y / z limit) for the others.

Tolerance, per element: |x - x64| <= C_ROUND * 2^-24 * K_eff * mag + aerr, with mag the same sum over magnitudes and K_eff the length of
the longest fp32 sum that feeds the element.  Rank positions, elite masks, the clip / no-clip choice of ClipUp and the NaN edges are
compared exactly.
"""

import math
import os

import numpy as np
import pytest
import torch

from oracle import es_oracle as O
from oracle import functional_oracle as FO

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import ops
    from evotorch_b200.algorithms import functional as F

DEV = "cuda"
EPS32 = 2.0**-24
F32 = np.float32
C_ROUND = 2.0
BIG = 70000  # more items than one launch's grid y / z holds (65535)
RANKINGS = ["centered", "linear", "nes", "normalized", "raw"]


def C(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def _check(name, got, ref, bound):
    """|got - ref| <= bound where ref is finite; NaN exactly where ref is NaN, equal infinities."""
    got, ref, bound = (np.asarray(v, np.float64) for v in (got, ref, bound))
    got, bound = np.broadcast_to(got, ref.shape), np.broadcast_to(bound, ref.shape)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{name}: NaN at {np.argwhere(np.isnan(got) != nan)[:5].tolist()}"
    inf = np.isinf(ref)
    assert np.array_equal(got[inf], ref[inf]), f"{name}: infinities differ"
    fin = ~(nan | inf)
    err = np.abs(got[fin] - ref[fin])
    r = float(np.max(err / bound[fin])) if err.size else 0.0
    assert r <= 1.0, f"{name}: error / bound = {r:.3g}"


def _probe_items(B, rng, extra=8):
    """first, last, both sides of 65535 and of each 256-item launch boundary that exists, plus a few random items"""
    cand = {0, B - 1, 255, 256, 257, 65534, 65535, 65536}
    cand |= set(rng.integers(0, B, extra).tolist())
    return sorted(i for i in cand if 0 <= i < B)


# ------------------------------------------------------------------------------------------------ K1 evok_sample_batched
@pytest.mark.parametrize("B", [1, 5, 255, 256, 257, BIG])
@pytest.mark.parametrize("D", [1, 3, 5, 4, 1024])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("shared", [True, False])
def test_sample_batched_follows_philox_per_item(B, D, symmetric, shared):
    """Item b draws from Philox stream stream_id0 + b: bit for bit the single-search sampler at that stream, and within the sampler's
    tolerance of `philox_population`, for the first and last items, both sides of 65535 and random ones; every item differs."""
    rng = np.random.default_rng(B * 31 + D * 7 + symmetric * 2 + shared)
    n = 4
    seed, sid0 = 0x5EED_0000_1234 + D, 11
    rows = 1 if shared else B
    mu = rng.uniform(-2, 2, (rows, D)).astype(np.float32)
    sg = rng.uniform(0.5, 1.5, (rows, D)).astype(np.float32)
    X = torch.empty(B, n, D, device=DEV)
    ops.sample_batched(X, C(mu[0]) if shared else C(mu), C(sg[0]) if shared else C(sg), symmetric=symmetric, seed=seed, stream_id0=sid0)
    for b in _probe_items(B, rng):
        m, s = mu[0 if shared else b], sg[0 if shared else b]
        ref = torch.empty(n, D, device=DEV)
        ops.sample_eval(ops.OBJ_NONE, ref, C(m), C(s), n_rows=n, symmetric=symmetric, seed=seed, stream_id=sid0 + b)
        assert torch.equal(X[b], ref), f"item {b}"
        np.testing.assert_allclose(N(X[b]), O.philox_population(m, s, n, symmetric, seed, sid0 + b), rtol=0, atol=3e-5 * float(s.max()) + 1e-6)
    fp = (X.view(B, -1).double() * torch.rand(n * D, dtype=torch.float64, device=DEV)).sum(1)
    assert torch.unique(fp).numel() == B


# ------------------------------------------------------------------------------------------------ K3 evok_rank_batched & co.
def _fitness_items(B, n, rng):
    """(B, n) fitnesses with ties, +-0 and, in item 1 / 2, +-inf / NaN"""
    f = np.round(rng.standard_normal((B, n)) * 4) / 4
    f[0, : min(n, 4)] = [0.0, -0.0, 0.0, -0.0][: min(n, 4)]
    if B > 1 and n >= 4:
        f[1, [1, n - 1]] = [np.inf, -np.inf]
    if B > 2 and n >= 4:
        f[2, [0, n // 2]] = np.nan
    return f.astype(np.float32)


RANK_SHAPES = [(2, 3), (1024, 3), (1025, 3), (8192, 3), (8193, 3), (20000, 2), (2, BIG), (16, BIG)]


@pytest.mark.parametrize("n,B", RANK_SHAPES)
@pytest.mark.parametrize("method", RANKINGS)
@pytest.mark.parametrize("maximize", [False, True])
def test_rank_batched_matches_the_oracle(n, B, method, maximize):
    """Utilities of every item: the oracle's ranking exactly for centered / linear / raw (stable order on ties, +-0 equal, NaN the
    largest), within rounding for nes and normalized (NaN where the item holds NaN or infinities of both signs)."""
    rng = np.random.default_rng(n * 13 + B + RANKINGS.index(method) * 2 + maximize)
    f = _fitness_items(B, n, rng)
    w = N(ops.rank_batched(C(f), method, maximize))
    for b in (range(B) if B <= 5 else _probe_items(B, rng)):
        ref = O.rank(f[b], method, maximize).astype(np.float64)
        if method in ("centered", "linear", "raw"):
            np.testing.assert_array_equal(w[b], ref, err_msg=f"item {b}")
        elif method == "nes":
            # the oracle sums the utility table in fp32 (pairwise), the kernel in float64: K_eff ~ log2(N)
            _check(f"nes item {b}", w[b], ref, C_ROUND * EPS32 * 32 * (np.abs(ref) + 1.0 / n))
        else:
            _check(f"normalized item {b}", w[b], ref, C_ROUND * EPS32 * 32 * (np.abs(ref) + 1.0))


ELITE_SHAPES = [(2, 3), (1024, 3), (8192, 3), (8193, 3), (20000, 2), (16, BIG)]


@pytest.mark.parametrize("n,B", ELITE_SHAPES)
@pytest.mark.parametrize("which", ["zero", "one", "all"])
def test_elite_mask_batched_and_weights_adjust_batched(n, B, which):
    """The elite mask marks exactly the num_elites largest weights of each item (stable on ties); weights_adjust mode 1 subtracts the
    item's mean, mode 2 divides by its sum of magnitudes."""
    rng = np.random.default_rng(n + B + len(which))
    w = (np.round(rng.standard_normal((B, n)) * 8) / 8).astype(np.float32)
    E = {"zero": 0, "one": 1, "all": n}[which]
    mask = N(ops.elite_mask_batched(C(w), E))
    items = range(B) if B <= 5 else _probe_items(B, rng)
    for b in items:
        ref = np.zeros(n, np.float32)
        ref[O.argsort_for_ranking(w[b], higher_is_better=False)[:E]] = 1
        np.testing.assert_array_equal(mask[b], ref, err_msg=f"item {b}")
    for mode in (1, 2):
        t = C(w)
        ops.weights_adjust_batched_(t, mode)
        got = N(t)
        for b in items:
            w64 = w[b].astype(np.float64)
            if mode == 1:
                ref, bound = w64 - w64.mean(), C_ROUND * EPS32 * (np.abs(w64) + 2 * abs(w64.mean()))
            else:
                ref = w64 / np.abs(w64).sum()
                bound = C_ROUND * EPS32 * 2 * np.abs(ref)
            _check(f"adjust{mode} item {b}", got[b], ref, bound + 1e-30)


# ------------------------------------------------------------------------------------------------ K4 evok_grad_batched
FORMS = [ops.GRAD_SEPARABLE, ops.GRAD_SYMMETRIC, ops.GRAD_EXP, ops.GRAD_MOMENTS] if torch.cuda.is_available() else [0, 1, 2, 3]
GRAD_SHAPES = [(3, 64, 8), (2, 0, 8), (2, 3000, 1024), (600, 32, 36), (5, 40, 7), (400, 16, 37), (BIG, 4, 4)]  # (items, n_rows, D)


@pytest.mark.parametrize("B,n,D", GRAD_SHAPES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("shared", [True, False])
def test_grad_batched_matches_float64(B, n, D, form, shared):
    """S1 / S2 of every form for few items (the single-item chunk plan), many items (one chunk each), > 65535 items, n = 0 (zeros),
    on the float4 path (D % 4 == 0) and the scalar one, with shared and per-item mu / sigma."""
    rng = np.random.default_rng(B + n * 3 + D * 5 + form * 7 + shared)
    rows = 1 if shared else B
    mu = rng.uniform(-1, 1, (rows, D)).astype(np.float32)
    sg = rng.uniform(0.5, 1.5, (rows, D)).astype(np.float32)
    X = (rng.standard_normal((B, n, D)) * 1.3 + rng.uniform(-1, 1, (B, 1, D))).astype(np.float32)
    w = (rng.standard_normal((B, n)) if form != ops.GRAD_MOMENTS else (rng.random((B, n)) < 0.3)).astype(np.float32)
    s_mu, s_sig = 0.37, 1.9
    if n == 0:  # an empty tensor has no data pointer: call the library with valid ones and n_rows = 0 (the memset path)
        from evotorch_b200 import _native as nat

        buf = torch.zeros(B * D + 4, device=DEV)
        g1, g2 = torch.full((B, D), np.nan, device=DEV), torch.full((B, D), np.nan, device=DEV)
        ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
        nat.check(nat.lib().evok_grad_batched(form, buf.data_ptr(), 0, D, buf.data_ptr(), C(mu).data_ptr(), 0 if shared else D, C(sg).data_ptr(),
                                              0 if shared else D, B, 0, D, s_mu, s_sig, g1.data_ptr(), g2.data_ptr(), ws.data_ptr(), ws.numel(),
                                              nat.stream_of(buf)), "evok_grad_batched")
        assert not N(g1).any() and not N(g2).any()
        return
    g1, g2 = ops.grad_batched(form, C(X), C(w), C(mu[0]) if shared else C(mu), C(sg[0]) if shared else C(sg), s_mu, s_sig)
    g1, g2 = N(g1), N(g2)
    k_eff = (n // 2 if form == ops.GRAD_SYMMETRIC else n) + 6
    for b in (range(B) if B <= 5 else _probe_items(B, rng)):
        m, s = mu[0 if shared else b], sg[0 if shared else b]
        ref = FO.weighted_sums(form, X[b], w[b], m, s)
        _check(f"s1 item {b}", g1[b], s_mu * ref["s1"], C_ROUND * EPS32 * k_eff * s_mu * ref["s1_mag"] + 1e-30)
        _check(f"s2 item {b}", g2[b], s_sig * ref["s2"], C_ROUND * EPS32 * k_eff * s_sig * ref["s2_mag"] + 1e-30)


# ------------------------------------------------------------------------------------------------ K5 evok_clipup_batched
@pytest.mark.parametrize("B", [255, 256, 257, 513])
@pytest.mark.parametrize("D", [1, 1023, 1024, 1025, 5000])
def test_clipup_batched_per_item_hyper_parameters(B, D):
    """Each item with its own (lr, momentum, max_speed): half the items clip, half do not (speed at least 25 % away from the limit);
    the velocity and centre of every item within rounding of `es_oracle.ClipUp`."""
    rng = np.random.default_rng(B * 3 + D)
    g = rng.standard_normal((B, D)).astype(np.float32)
    v0 = (rng.standard_normal((B, D)) * 0.1 / math.sqrt(D)).astype(np.float32)
    c0 = rng.uniform(-1, 1, (B, D)).astype(np.float32)
    lr = rng.uniform(0.05, 0.5, B)
    mom = rng.uniform(0.0, 0.95, B)
    speed = np.array([np.linalg.norm(mom[b] * v0[b].astype(np.float64) + lr[b] * g[b] / np.linalg.norm(g[b].astype(np.float64)))
                      for b in range(B)])
    cap = np.where(np.arange(B) % 2 == 0, speed * 0.75, speed * 1.25)
    vel, cen = C(v0), C(c0)
    ops.clipup_batched_(C(g), vel, cen, lr.tolist(), mom.tolist(), cap.tolist())
    vel, cen = N(vel), N(cen)
    for b in range(B):
        lr_b, mom_b = F32(lr[b]), F32(mom[b])
        r = FO.clipup_tell(c0[b], v0[b], g[b], lr=lr_b, momentum=mom_b, max_speed=F32(cap[b]))
        assert r["clipped"] == (b % 2 == 0)
        g64 = g[b].astype(np.float64)
        mag = mom_b * np.abs(v0[b]) + lr_b * np.abs(g64) / np.linalg.norm(g64)  # the terms of the new velocity, before the clip
        bound = C_ROUND * EPS32 * (4 * mag + 4 * np.abs(r["velocity"])) + 1e-30
        _check(f"velocity item {b}", vel[b], r["velocity"], bound)
        _check(f"center item {b}", cen[b], r["center"], bound + C_ROUND * EPS32 * (np.abs(c0[b]) + np.abs(r["center"])))


# ------------------------------------------------------------------------------------------------ K5 sigma updates
def _sigma_case(B, D, rng, with_bounds):
    s = rng.uniform(0.2, 2.0, (B, D)).astype(np.float32)
    s[:, 0] = 0.0  # sigma = 0 with max_change = inf: the allowed change is NaN
    g = rng.standard_normal((B, D)).astype(np.float32)
    g[:, 1] = np.nan  # a NaN target
    if not with_bounds:
        return s, g, None, None, None
    lb = np.full((B, D), 0.3, np.float32)
    ub = np.full((B, D), 1.6, np.float32)
    mc = np.full((B, D), 0.2, np.float32)
    mc[:, 0] = np.inf
    mc[:, 2] = np.inf
    lb[:, 3] = 0.0
    return s, g, lb, ub, mc


@pytest.mark.parametrize("B", [3, 300])
@pytest.mark.parametrize("exp_form", [False, True])
@pytest.mark.parametrize("bounds", ["none", "all", "lb_only"])
def test_sigma_update_batched_matches_modify_tensor(B, exp_form, bounds):
    """sigma <- clamp(target) with per-item learning rates over the 256-item launch boundary, NaN where torch gives NaN: a NaN target,
    and sigma = 0 with max_change = inf (|0| * inf = NaN through torch.max / torch.min)."""
    rng = np.random.default_rng(B + exp_form * 2 + len(bounds))
    D = 37
    s, g, lb, ub, mc = _sigma_case(B, D, rng, bounds != "none")
    if bounds == "lb_only":
        ub = mc = None
    lr = rng.uniform(0.05, 0.5, B)
    t = C(s)
    ops.sigma_update_batched_(t, C(g), lr.tolist(), exp_form, lb=None if lb is None else C(lb), ub=None if ub is None else C(ub),
                              max_change=None if mc is None else C(mc))
    got = N(t)
    for b in range(B):
        ref, target = FO.sigma_update(s[b], g[b], float(np.float32(lr[b])), exp_form=exp_form, stdev_min=None if lb is None else lb[b],
                                      stdev_max=None if ub is None else ub[b], stdev_max_change=None if mc is None else mc[b])
        step = np.abs(lr[b] * g[b].astype(np.float64))
        bound = C_ROUND * EPS32 * (np.abs(target) * (4 + step) if exp_form else np.abs(s[b]) + 2 * step) + 1e-30
        _check(f"sigma item {b}", got[b], ref, bound)
        if mc is not None:
            assert np.isnan(got[b, 0])


@pytest.mark.parametrize("kind", ["none", "scalar", "vector"])
@pytest.mark.parametrize("exp_form", [False, True])
def test_sigma_update_single_matches_modify_tensor(kind, exp_form):
    """The per-item kernel: scalar bounds (NaN = not set), vector bounds (a NaN entry is data and gives NaN), sigma = 0 with an
    infinite max change."""
    rng = np.random.default_rng(len(kind) + exp_form)
    D = 1029
    s, g, lb, ub, mc = _sigma_case(1, D, rng, True)
    s, g = s[0], g[0]
    if kind == "none":
        args, oargs = {}, {}
    elif kind == "scalar":
        args = dict(lb=0.3, ub=float("nan"), max_change=float("inf"))
        oargs = dict(stdev_min=0.3, stdev_max=None, stdev_max_change=np.inf)
    else:
        lb, ub, mc = lb[0], ub[0], mc[0]
        lb[5] = np.nan
        args = dict(lb=C(lb), ub=C(ub), max_change=C(mc))
        oargs = dict(stdev_min=lb, stdev_max=ub, stdev_max_change=mc)
    t = C(s)
    ops.sigma_update_(t, C(g), 0.3, exp_form, **args)
    ref, target = FO.sigma_update(s, g, 0.3, exp_form=exp_form, **oargs)
    step = np.abs(0.3 * g.astype(np.float64))
    _check("sigma", N(t), ref, C_ROUND * EPS32 * (np.abs(target) * (4 + step) if exp_form else np.abs(s) + 2 * step) + 1e-30)
    if kind != "none":
        assert np.isnan(N(t)[0])
    if kind == "vector":
        assert np.isnan(N(t)[5])


# ------------------------------------------------------------------------------------------------ K5 evok_cem_finalize
@pytest.mark.parametrize("E", [0, 1, 2, 40])
@pytest.mark.parametrize("offset", [0.0, 30.0])
def test_cem_finalize_from_the_batched_moments(E, offset):
    """Elite moments by grad_batched(MOMENTS) with the elite mask, then cem_finalize, against the two-pass float64 mean and std: E = 0
    gives NaN for both, E = 1 a NaN std (as torch.std), E >= 2 within the one-pass bound, also with the elites 30 spreads from mu
    (the cancellation in S2 - S1^2 / E)."""
    rng = np.random.default_rng(E * 2 + int(offset))
    B, n, D = 3, 40, 1000
    mu = rng.uniform(-1, 1, (B, D)).astype(np.float32)
    sg = rng.uniform(0.5, 1.5, (B, D)).astype(np.float32)
    X = (mu[:, None] + offset + rng.standard_normal((B, n, D))).astype(np.float32)
    f = rng.standard_normal((B, n)).astype(np.float32)
    w = ops.rank_batched(C(f), "raw", False)
    mask = ops.elite_mask_batched(w, E)
    s1, s2 = ops.grad_batched(ops.GRAD_MOMENTS, C(X), mask, C(mu), C(sg), 1.0, 1.0)
    gm, gs = ops.cem_finalize(s1.view(-1), s2.view(-1), C(sg).view(-1), E)
    gm, gs = N(gm).reshape(B, D), N(gs).reshape(B, D)
    for b in range(B):
        r = FO.cem_moments(X[b], f[b], mu[b], parenthood_ratio=E / n, maximize=False)
        assert r["num_elites"] == E
        if E == 0:
            assert np.isnan(gm[b]).all() and np.isnan(gs[b]).all()
            continue
        k = E + 6
        _check(f"grad_mu item {b}", gm[b], r["mean"] - mu[b], C_ROUND * EPS32 * (k * r["s1_mag"] / E + np.abs(r["mean"] - mu[b])) + 1e-30)
        if E == 1:
            assert np.isnan(gs[b]).all()
            continue
        var_err = C_ROUND * EPS32 * k * (r["s2"] + r["s1"] ** 2 / E) / (E - 1)
        std32 = gs[b].astype(np.float64) + sg[b]
        _check(f"std item {b}", std32, r["std"], var_err / (std32 + r["std"]) + C_ROUND * EPS32 * (r["std"] + sg[b]))


def test_cem_finalize_nan_variance_stays_nan():
    """A NaN moment gives a NaN std (torch.clamp_min keeps NaN), a negative rounding residue gives 0."""
    s1 = C([np.nan, 1.0, 2.0])
    s2 = C([1.0, np.nan, 1.9999])  # item 3: S2 - S1^2 / E < 0 by rounding
    sg = C([0.5, 0.5, 0.5])
    gm, gs = ops.cem_finalize(s1, s2, sg, 2)
    gs = N(gs)
    assert np.isnan(gs[0]) and np.isnan(gs[1]) and gs[2] == -0.5
    assert np.isnan(N(gm)[0])


# ------------------------------------------------------------------------------------------------ K5 adam / sgd / axpy
@pytest.mark.parametrize("t", [1, 10000])
@pytest.mark.parametrize("outputs", ["both", "step_out", "mu", "none"])
def test_adam_step_matches_the_oracle(t, outputs):
    rng = np.random.default_rng(t + len(outputs))
    D = 1031
    g = rng.standard_normal(D).astype(np.float32)
    m0 = (rng.standard_normal(D) * 0.1 * (t > 1)).astype(np.float32)
    v0 = (rng.random(D) * 0.5 * (t > 1)).astype(np.float32)
    c0 = rng.uniform(-1, 1, D).astype(np.float32)
    m, v, mu, so = C(m0), C(v0), C(c0), torch.full((D,), np.nan, device=DEV)
    ops.adam_step(C(g), m, v, t, 0.01, 0.9, 0.999, 1e-8, step_out=so if outputs in ("both", "step_out") else None,
                  mu=mu if outputs in ("both", "mu") else None)
    # the kernel receives the betas as fp32 (the C ABI): 1 - beta2 of fp32(0.999) differs from fp32(1 - 0.999) by 1.3e-5 relative
    r = FO.adam_tell(c0, m0, v0, t - 1, g, lr=F32(0.01), beta1=F32(0.9), beta2=F32(0.999), epsilon=F32(1e-8))
    _check("m", N(m), r["m"], C_ROUND * EPS32 * 2 * (np.abs(m0) + np.abs(g)) + 1e-30)
    _check("v", N(v), r["v"], C_ROUND * EPS32 * 3 * (np.abs(v0) + g.astype(np.float64) ** 2) + 1e-30)
    # the step is relative to m, which cancels where b1 m0 and (1 - b1) g have opposite signs: scale by the magnitude of its terms
    b1, b2 = float(F32(0.9)), float(F32(0.999))
    m_mag = b1 * np.abs(m0) + (1 - b1) * np.abs(g)
    step_mag = 0.01 / (1 - b1**t) * m_mag / (np.sqrt(r["v"] / (1 - b2**t)) + 1e-8)
    step_bound = C_ROUND * EPS32 * 8 * (np.abs(r["step"]) + step_mag) + 1e-30
    if outputs in ("both", "step_out"):
        _check("step", N(so), r["step"], step_bound)
    else:
        assert torch.isnan(so).all()
    if outputs in ("both", "mu"):
        _check("mu", N(mu), r["center"], step_bound + C_ROUND * EPS32 * np.abs(r["center"]))
    else:
        assert np.array_equal(N(mu), c0)


@pytest.mark.parametrize("momentum", [0.0, 0.7])
@pytest.mark.parametrize("first_step", [True, False])
@pytest.mark.parametrize("outputs", ["both", "step_out", "mu"])
def test_sgd_step_and_axpy_match_the_oracle(momentum, first_step, outputs):
    """buf <- momentum buf + g (first step: buf = g), step = lr buf; momentum 0 runs without a buffer.  axpy: mu += lr g."""
    rng = np.random.default_rng(int(momentum * 10) + first_step * 3 + len(outputs))
    D, lr = 1500, 0.05
    g = rng.standard_normal(D).astype(np.float32)
    b0 = rng.standard_normal(D).astype(np.float32)
    c0 = rng.uniform(-1, 1, D).astype(np.float32)
    buf = C(b0) if momentum else None
    so, mu = torch.full((D,), np.nan, device=DEV), C(c0)
    ops.sgd_step(C(g), buf, first_step, lr, momentum, step_out=so if outputs != "mu" else None, mu=mu if outputs != "step_out" else None)
    # the functional form from velocity lr * b0: the same as es_oracle.SGD's buffer form (see functional_oracle.sgd_tell)
    prev = np.zeros(D) if (first_step or not momentum) else lr * b0.astype(np.float64)
    r = FO.sgd_tell(c0, prev, g, lr=lr, momentum=momentum)
    step = r["velocity"]
    bound = C_ROUND * EPS32 * 3 * (np.abs(step) + lr * np.abs(g) + lr * momentum * np.abs(b0)) + 1e-30
    if outputs != "mu":
        _check("step", N(so), step, bound)
    if outputs != "step_out":
        _check("mu", N(mu), r["center"], bound + C_ROUND * EPS32 * np.abs(r["center"]))
    else:
        assert np.array_equal(N(mu), c0)
    if momentum:
        _check("buf", N(buf), step / lr, C_ROUND * EPS32 * 3 * (np.abs(step / lr) + np.abs(g) + momentum * np.abs(b0)))
    a = C(c0)
    ops.axpy_(a, C(g), -0.3)
    _check("axpy", N(a), c0.astype(np.float64) - 0.3 * g, C_ROUND * EPS32 * 2 * (np.abs(c0) + 0.3 * np.abs(g)) + 1e-30)


# ------------------------------------------------------------------------------------------------ whole tells through the public API
@pytest.fixture(params=["batched", "loop"])
def tell_mode(request, monkeypatch):
    """the default one-launch-per-stage tells, and the per-item launch chains of EVOTORCH_B200_FUNCTIONAL_LOOP=1"""
    monkeypatch.setenv("EVOTORCH_B200_FUNCTIONAL_LOOP", "1" if request.param == "loop" else "0")
    return request.param


def _population(center, stdev, n, symmetric, rng):
    Z = rng.standard_normal(center.shape[:-1] + (n // 2 if symmetric else n, center.shape[-1]))
    if symmetric:
        X = np.empty(center.shape[:-1] + (n, center.shape[-1]))
        X[..., 0::2, :], X[..., 1::2, :] = center[..., None, :] + stdev[..., None, :] * Z, center[..., None, :] - stdev[..., None, :] * Z
    else:
        X = center[..., None, :] + stdev[..., None, :] * Z
    return X.astype(np.float32)


def _pgpe_tell_case(opt, ranking, symmetric, sense, batch, rng, *, shared_center=False, shared_stdev=False, n=16, D=6):
    """One pgpe_tell on CUDA against the oracle, item by item; returns nothing, asserts."""
    full = batch if batch else ()
    center0 = rng.uniform(-2, 2, (() if shared_center else full) + (D,)).astype(np.float32)
    stdev0 = rng.uniform(0.6, 1.4, (() if shared_stdev else full) + (D,)).astype(np.float32)
    nb = int(np.prod(full)) if full else 1
    lrs = np.float32(rng.uniform(0.05, 0.3, nb)).astype(np.float64)
    lr_t = torch.as_tensor(lrs.reshape(full) if full else lrs[0], dtype=torch.float32)
    opt_cfg = {"clipup": dict(momentum=0.8, max_speed=lr_t * 2.0), "adam": dict(beta1=0.85), "sgd": dict(momentum=0.6)}[opt]
    state = F.pgpe(center_init=C(center0), center_learning_rate=lr_t, stdev_learning_rate=0.15, objective_sense=sense, ranking_method=ranking,
                   optimizer=opt, optimizer_config=opt_cfg, stdev_init=C(stdev0), stdev_min=0.5, stdev_max=1.5, stdev_max_change=0.25,
                   symmetric=symmetric)
    X = _population(np.broadcast_to(center0, full + (D,)), np.broadcast_to(stdev0, full + (D,)), n, symmetric, rng)
    f = (np.round((X.astype(np.float64) ** 2).sum(-1) * 4) / 4).astype(np.float32)
    new = F.pgpe_tell(state, C(X), C(f))
    got_c = N(new.optimizer_state.center).reshape(nb, D)
    got_s = N(new.stdev).reshape(nb, D)
    Xf, ff = X.reshape(nb, n, D), f.reshape(nb, n)
    cf, sf = np.broadcast_to(center0, full + (D,)).reshape(nb, D), np.broadcast_to(stdev0, full + (D,)).reshape(nb, D)
    k_eff = (n // 2 if symmetric else n) + 8
    for b in (range(nb) if nb <= 300 else _probe_items(nb, rng)):
        gr = FO.pgpe_gradients(Xf[b], ff[b], cf[b], sf[b], ranking_method=ranking, maximize=(sense == "max"), symmetric=symmetric)
        err_g = C_ROUND * EPS32 * k_eff * gr["mu_mag"]
        ref_s, target = FO.sigma_update(sf[b], gr["sigma"], 0.15, stdev_min=0.5, stdev_max=1.5, stdev_max_change=0.25)
        _check(f"stdev item {b}", got_s[b], ref_s,
               C_ROUND * EPS32 * (2 * np.abs(sf[b]) + 0.15 * k_eff * gr["sigma_mag"]) + 0.15 * C_ROUND * EPS32 * np.abs(gr["sigma"]))
        gnorm = np.linalg.norm(gr["mu"])
        if opt == "clipup":
            r = FO.clipup_tell(cf[b], np.zeros(D), gr["mu"], lr=lrs[b], momentum=0.8, max_speed=2.0 * lrs[b])
            sens = lrs[b] * (err_g + np.linalg.norm(err_g)) / gnorm
        elif opt == "adam":
            r = FO.adam_tell(cf[b], np.zeros(D), np.zeros(D), 0, gr["mu"], lr=lrs[b], beta1=F32(0.85), beta2=F32(0.999), epsilon=F32(1e-8))
            sens = lrs[b] * err_g * 1e-8 / gr["mu"] ** 2  # at t = 1 the step is lr g / (|g| + eps): d step / d g = lr eps / (|g| + eps)^2
            assert (np.abs(gr["mu"]) > 4 * err_g).all(), "a gradient component at rounding level: the sign of the Adam step is undecided"
        else:
            r = FO.sgd_tell(cf[b], np.zeros(D), gr["mu"], lr=lrs[b], momentum=0.6)
            sens = lrs[b] * err_g
        _check(f"center item {b}", got_c[b], r["center"], sens + C_ROUND * EPS32 * 8 * (np.abs(r["center"]) + np.abs(r["center"] - cf[b])) + 1e-30)


@pytest.mark.parametrize("opt", ["clipup", "adam", "sgd"])
@pytest.mark.parametrize("ranking", RANKINGS)
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("sense", ["min", "max"])
def test_pgpe_tell_every_configuration(opt, ranking, symmetric, sense, tell_mode):
    """Every optimizer x ranking x sampling x sense, on a (2, 3) batch with per-item learning rates."""
    rng = np.random.default_rng(["clipup", "adam", "sgd"].index(opt) * 40 + RANKINGS.index(ranking) * 4 + symmetric * 2 + (sense == "max"))
    _pgpe_tell_case(opt, ranking, symmetric, sense, (2, 3), rng)


@pytest.mark.parametrize("batch", [(), (1,), (3,), (2, 3), (300,), (BIG,)])
@pytest.mark.parametrize("layout", ["per_item", "shared_center", "shared_stdev"])
def test_pgpe_tell_batch_shapes_and_broadcasting(batch, layout, tell_mode):
    """Batch shapes from none to 70000 items (the last at N = 4, D = 3), a centre shared by batched values, a batched stdev with a
    shared centre, per-item learning rates."""
    if tell_mode == "loop" and batch == (BIG,):
        pytest.skip("the per-item launch chains of 70000 items are a timing matter, not a correctness one")
    if batch == () and layout != "per_item":
        pytest.skip("nothing to broadcast without a batch")
    rng = np.random.default_rng(len(batch) * 10 + sum(batch) + len(layout))
    small = batch == (BIG,)
    _pgpe_tell_case("clipup", "centered", True, "min", batch, rng, shared_center=(layout == "shared_center"),
                    shared_stdev=(layout == "shared_stdev"), n=4 if small else 16, D=3 if small else 6)


@pytest.mark.parametrize("batch", [(), (1,), (3,), (2, 3), (300,), (BIG,)])
@pytest.mark.parametrize("ratio", [0.1, 0.25, 1.0])
def test_cem_tell_batch_shapes(batch, ratio, tell_mode):
    """cem_tell on CUDA against the two-pass float64 elite moments; ratio 0.1 of N = 10 is the one-elite case (NaN stdev)."""
    if tell_mode == "loop" and batch == (BIG,):
        pytest.skip("the per-item launch chains of 70000 items are a timing matter, not a correctness one")
    rng = np.random.default_rng(len(batch) * 10 + sum(batch) + int(ratio * 100))
    n, D = (10, 3) if batch == (BIG,) else (10, 6)
    full = batch
    nb = int(np.prod(full)) if full else 1
    center0 = rng.uniform(-2, 2, full + (D,)).astype(np.float32)
    stdev0 = rng.uniform(0.6, 1.4, full + (D,)).astype(np.float32)
    st = F.cem(center_init=C(center0), parenthood_ratio=ratio, objective_sense="min", stdev_init=C(stdev0), stdev_min=0.2, stdev_max=3.0,
               stdev_max_change=0.5)
    X = _population(center0, stdev0, n, False, rng)
    f = (X.astype(np.float64) ** 2).sum(-1).astype(np.float32)
    new = F.cem_tell(st, C(X), C(f))
    got_c, got_s = N(new.center).reshape(nb, D), N(new.stdev).reshape(nb, D)
    Xf, ff, cf, sf = X.reshape(nb, n, D), f.reshape(nb, n), center0.reshape(nb, D), stdev0.reshape(nb, D)
    for b in (range(nb) if nb <= 300 else _probe_items(nb, rng)):
        r = FO.cem_tell(Xf[b], ff[b], cf[b], sf[b], parenthood_ratio=ratio, maximize=False, stdev_min=0.2, stdev_max=3.0, stdev_max_change=0.5)
        E = r["num_elites"]
        k = E + 6
        _check(f"center item {b}", got_c[b], r["center"], C_ROUND * EPS32 * (k * r["s1_mag"] / E + 2 * np.abs(r["center"])) + 1e-30)
        if E == 1:
            assert np.isnan(got_s[b]).all()
            continue
        var_err = C_ROUND * EPS32 * k * (r["s2"] + r["s1"] ** 2 / E) / (E - 1)
        _check(f"stdev item {b}", got_s[b], r["stdev"], var_err / (2 * r["std"]) + C_ROUND * EPS32 * 4 * (r["std"] + sf[b]))


@pytest.mark.parametrize("tag,kw", [("one_elite", dict(parenthood_ratio=0.03, objective_sense="min", stdev_init=1.0)),
                                    ("zero_elites", dict(parenthood_ratio=0.01, objective_sense="max", stdev_init=1.0)),
                                    ("zero_stdev", dict(parenthood_ratio=0.25, objective_sense="min"))])
def test_cem_tell_reproduces_the_reference_edges(tag, kw, tell_mode):
    """The reference's NaN edges (tests/golden/functional_golden.npz) in both tell modes: NaN exactly where the reference has NaN."""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "functional_golden.npz"))
    kw = dict(kw)
    if tag == "zero_stdev":
        kw["stdev_init"] = C(gold[f"cem/{tag}/stdev0"])
    st = F.cem(center_init=C(gold[f"cem/{tag}/center0"]), **kw)
    new = F.cem_tell(st, C(gold[f"cem/{tag}/values"][0]), C(gold[f"cem/{tag}/evals"][0]))
    for name, got in (("center", new.center), ("stdev", new.stdev)):
        want = gold[f"cem/{tag}/{name}"][0]
        np.testing.assert_array_equal(np.isnan(N(got)), np.isnan(want), err_msg=name)
        np.testing.assert_allclose(N(got), want, rtol=1e-5, atol=2e-5, equal_nan=True)
