"""Isolation of the kernels: a result depends only on the data inside its operands' logical extent.

Several kernels read past that extent on purpose (the aligned 128-bit loads of the policy forward, the TMA tiles of the GEMM, the
shifted gather of the shared-minibatch forward) and rely on multiplying the extra values by zero -- which breaks as soon as those
bytes hold Inf or NaN (Inf * 0 = NaN).  Every check here runs a kernel twice on the same data; the runs differ only in what sits
outside the logical extent (neighbouring parameter rows, row padding, rows past the end, rows whose weights are zero, workspace
contents), and their results must agree bit for bit.  The clean run is also compared with a float64 reference at the tolerances
the rest of the suite uses for that kernel.  Needs a CUDA device (H100): run with `-m gpu`."""

import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import _native as nat
    from evotorch_b200 import ops

DEV = "cuda"
NAN, INF = float("nan"), float("inf")
POISONS = (INF, -INF, NAN)
FILLS = (0.0, NAN, INF, -INF)  # what may sit outside the extent: the first is the clean run
FORMS = {"separable": 0, "symmetric": 1, "exp": 2, "moments": 3}


def embed(t: torch.Tensor, pad: int = 0, extra_rows: int = 0, fill: float = NAN) -> torch.Tensor:
    """A (rows, cols) view of `t` inside a (rows + extra_rows, cols + pad) buffer whose other elements are `fill`."""
    rows, cols = t.shape
    buf = torch.full((rows + extra_rows, cols + pad), fill, dtype=t.dtype, device=t.device)
    buf[:rows, :cols] = t
    return buf[:rows, :cols]


def outside(view: torch.Tensor, pad: int, extra_rows: int = 0) -> torch.Tensor:
    """The elements of the buffer behind `embed(...)` that lie outside `view` (row padding and the rows past the end)."""
    rows, cols = view.shape
    full = view.as_strided((rows + extra_rows, cols + pad), (view.stride(0), 1))
    mask = torch.ones_like(full, dtype=torch.bool)
    mask[:rows, :cols] = False
    return full[mask]


def assert_untouched(view, pad, extra_rows=0, fill=NAN):
    rest = outside(view, pad, extra_rows)
    if math.isnan(fill):
        assert bool(torch.isnan(rest).all()), "the kernel wrote outside its output's extent"
    else:
        assert bool((rest == fill).all()), "the kernel wrote outside its output's extent"


def rel_err(got: torch.Tensor, ref: torch.Tensor) -> float:
    return float((got.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ K8 per-policy forward
MLP_NETS = [
    ((376, 256, 17), ("tanh", "none")),  # L = 100 881 (odd): rows at all four 16-byte phases
    ((8, 512, 2), ("none", "tanh")),
    ((12, 16, 4), ("relu", "none")),
    ((33, 70, 9, 4), ("relu", "sigmoid", "tanh")),  # scalar layer 0
    ((33, 64, 8, 4), ("tanh", "relu", "none")),  # scalar layer 0, vector layers 1 and 2
]
ACT64 = {"tanh": torch.tanh, "relu": torch.relu, "sigmoid": torch.sigmoid, "none": lambda t: t}


def mlp_length(dims):
    return sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))


def mlp_ref(P, X, dims, acts):
    """float64 vmap(functional_call) of the flat torch.nn.Linear parameter rows: row i of P applied to row i of X."""
    n = P.shape[0]
    h = X.double()
    off = 0
    for l, act in enumerate(acts):
        W = P[:, off:off + dims[l] * dims[l + 1]].double().reshape(n, dims[l + 1], dims[l])
        off += dims[l] * dims[l + 1]
        b = P[:, off:off + dims[l + 1]].double()
        off += dims[l + 1]
        h = ACT64[act](torch.einsum("noi,ni->no", W, h) + b)
    return h


def prep_ref(X, s, ss, count, min_var, lo, hi):
    mean = s.double() / count
    var = torch.clamp(ss.double() / count - mean * mean, min=min_var)
    return torch.clamp((X.double() - mean) / var.sqrt(), lo, hi)


N_POL = 11  # rows 1 .. 9 are interior rows (vector path) and cover every 16-byte phase


def _mlp_problem(dims, seed):
    g = gen(seed)
    L = mlp_length(dims)
    P = torch.randn(N_POL, L, device=DEV, generator=g) * 0.1
    X = torch.randn(N_POL, dims[0], device=DEV, generator=g)
    return P, X, L


@pytest.mark.parametrize("dims,acts", MLP_NETS)
@pytest.mark.parametrize("pad", [0, 1, 2, 3, 4])
def test_mlp_forward_ignores_neighbour_rows_and_padding(dims, acts, pad):
    P, X, L = _mlp_problem(dims, len(dims) * 100 + pad)
    O = dims[-1]
    ref = mlp_ref(P, X, dims, acts)
    params, obs = embed(P, pad, 1), embed(X, pad, 1)
    out = embed(torch.zeros(N_POL, O, device=DEV), pad, 1)
    clean = ops.mlp_forward(params, obs, dims, acts, out=out).clone()
    assert_untouched(out, pad, 1)
    torch.testing.assert_close(clean.double(), ref, rtol=2e-5, atol=2e-5)
    # the same data in zero padding: bit-identical
    z = ops.mlp_forward(embed(P, pad, 1, 0.0), embed(X, pad, 1, 0.0), dims, acts)
    assert torch.equal(z, clean)
    # one poisoned row at a time: every other row keeps its bits
    for r in range(1, 7):  # interior rows; their successors 2 .. 7 cover every phase
        for v in POISONS:
            for what in ("row", "tail"):
                saved = params[r].clone()
                if what == "row":
                    params[r] = v
                else:
                    params[r, L - 4:] = v  # the last floats of the row: the last layer's biases
                got = ops.mlp_forward(params, obs, dims, acts)
                params[r] = saved
                keep = torch.arange(N_POL, device=DEV) != r
                bad = [i for i in range(N_POL) if i != r and not torch.equal(got[i], clean[i])]
                assert not bad, f"row {r} = {v} ({what}) changed rows {bad} (phase of row {r + 1}: {((r + 1) * params.stride(0)) % 4})"
                assert torch.equal(got[keep], clean[keep])


@pytest.mark.parametrize("dims,acts", MLP_NETS)
@pytest.mark.parametrize("pad", [0, 1, 4])
def test_mlp_forward_prep_ignores_inactive_poisoned_rows(dims, acts, pad):
    P, X, L = _mlp_problem(dims, len(dims) * 1000 + pad)
    g = gen(pad + 7)
    s = torch.randn(dims[0], device=DEV, generator=g) * 3
    ss = s * s / 5 + torch.rand(dims[0], device=DEV, generator=g) * 4 + 0.5
    count = torch.tensor([5], dtype=torch.int64, device=DEV)
    kw = dict(obs_sum=s, obs_sumsq=ss, obs_count=count, min_variance=1e-2, clip=(-2.0, 2.0))
    bad_rows = [2, 3, 7]
    active = torch.ones(N_POL, dtype=torch.bool, device=DEV)
    active[bad_rows] = False
    params, obs = embed(P, pad, 1), embed(X, pad, 1)
    out = embed(torch.zeros(N_POL, dims[-1], device=DEV), pad, 1)
    clean = ops.mlp_forward(params, obs, dims, acts, out=out, active=active, **kw).clone()
    assert_untouched(out, pad, 1)
    ref = mlp_ref(P, prep_ref(X, s, ss, 5.0, 1e-2, -2.0, 2.0), dims, acts)
    ref[~active] = 0.0
    torch.testing.assert_close(clean.double(), ref, rtol=1e-4, atol=1e-5)
    assert int(torch.count_nonzero(clean[~active])) == 0
    for v in POISONS:
        params[bad_rows] = v
        obs[bad_rows] = v
        got = ops.mlp_forward(params, obs, dims, acts, active=active, **kw)
        assert torch.equal(got, clean), f"poison {v}"
        assert bool((got[~active] == 0).all()) and not bool(torch.signbit(got[~active]).any())
        params[bad_rows] = P[bad_rows]
        obs[bad_rows] = X[bad_rows]


# ------------------------------------------------------------------------------------------------ shared-minibatch forward
@pytest.mark.parametrize("dims,acts,n,B", [((376, 256, 17), ("tanh", "none"), 12, 70), ((6, 16, 3), ("relu", "none"), 10, 256),
                                           ((33, 40, 24, 5), ("tanh", "sigmoid", "none"), 13, 31), ((8, 512, 2), ("none", "tanh"), 9, 40)])
def test_mlp_forward_shared_ignores_neighbour_rows(dims, acts, n, B):
    g = gen(n * B)
    L = mlp_length(dims)
    P = torch.randn(n, L, device=DEV, generator=g) * 0.3
    x = torch.randn(B, dims[0], device=DEV, generator=g)
    clean = ops.mlp_forward_shared(P, x, dims, acts)
    h = x.double().unsqueeze(0).expand(n, B, dims[0])
    off = 0
    for l in range(len(acts)):
        W = P[:, off:off + dims[l] * dims[l + 1]].double().view(n, dims[l + 1], dims[l])
        off += dims[l] * dims[l + 1]
        b = P[:, off:off + dims[l + 1]].double()
        off += dims[l + 1]
        h = ACT64[acts[l]](torch.einsum("nbi,noi->nbo", h, W) + b[:, None, :])
    assert float((clean.double() - h).abs().max()) <= 2e-5 * max(float(h.abs().max()), 1.0)
    for r in (1, 2, 3, 4, n - 1):
        for v in POISONS:
            Pp = P.clone()
            Pp[r] = v
            got = ops.mlp_forward_shared(Pp, x, dims, acts)
            bad = [i for i in range(n) if i != r and not torch.equal(got[i], clean[i])]
            assert not bad, f"row {r} = {v} changed rows {bad}"
            Pp = P.clone()
            Pp[r, L - 3:] = v
            got = ops.mlp_forward_shared(Pp, x, dims, acts)
            bad = [i for i in range(n) if i != r and not torch.equal(got[i], clean[i])]
            assert not bad, f"last floats of row {r} = {v} changed rows {bad}"


# ------------------------------------------------------------------------------------------------ K2 evaluation
@pytest.mark.parametrize("objective", ["sphere", "rastrigin", "ackley"])
@pytest.mark.parametrize("D", [64, 37])
@pytest.mark.parametrize("pad", [1, 2, 3, 4])
def test_evaluate_ignores_padding(objective, D, pad):
    n = 67
    X = torch.randn(n, D, device=DEV, generator=gen(D + pad)) * 2.5
    X64 = X.double()
    if objective == "sphere":
        ref = (X64**2).sum(1)
    elif objective == "rastrigin":
        ref = 10.0 * D + (X64**2 - 10.0 * torch.cos(2 * math.pi * X64)).sum(1)
    else:
        ref = -20 * torch.exp(-0.2 * torch.sqrt((X64**2).mean(1))) - torch.exp(torch.cos(2 * math.pi * X64).mean(1)) + 20 + math.e
    runs = [ops.evaluate(ops.OBJECTIVE_IDS[objective], embed(X, pad, 2, fill)) for fill in FILLS]
    torch.testing.assert_close(runs[0].double(), ref, rtol=2e-6 * math.sqrt(D) + 2e-6, atol=2e-5)
    for fill, got in zip(FILLS[1:], runs[1:]):
        assert torch.equal(got, runs[0]), f"padding {fill}"


# ------------------------------------------------------------------------------------------------ K4 gradient
def grad_ref(form, X, w, mu, sg, scale_mu, scale_sigma):
    """float64 restatement of the four gradient forms; also returns the absolute-value sums that set the tolerance."""
    X64, w64, mu64, sg64 = X.double(), w.double(), mu.double(), sg.double()
    if form == "symmetric":
        eps = X64[0::2] - mu64
        a, b = (w64[0::2] - w64[1::2]) / 2, (w64[0::2] + w64[1::2]) / 2
        g = (eps**2 - sg64**2) / sg64
    else:
        eps = X64 - mu64
        a = b = w64
        g = {"separable": (eps**2 - sg64**2) / sg64, "exp": (eps / sg64) ** 2 - 1, "moments": eps**2}[form]
    keep_a, keep_b = a != 0, b != 0  # zero-weight rows take no part (their values may be non-finite)
    ea = torch.where(keep_a[:, None], eps, 0.0)
    gb = torch.where(keep_b[:, None], g, 0.0)
    ref_m = scale_mu * (a[:, None] * ea).sum(0)
    ref_s = scale_sigma * (b[:, None] * gb).sum(0)
    tol_m = 3e-6 * abs(scale_mu) * float((a.abs()[:, None] * ea.abs()).sum(0).max()) + 1e-9
    tol_s = 3e-6 * abs(scale_sigma) * float((b.abs()[:, None] * (gb.abs() + 1)).sum(0).max()) + 1e-9
    return ref_m, ref_s, tol_m, tol_s


def _grad_data(n, D, seed, form):
    g = gen(seed)
    mu = torch.randn(D, device=DEV, generator=g)
    sg = torch.rand(D, device=DEV, generator=g) * 0.5 + 0.2
    X = mu + sg * torch.randn(n, D, device=DEV, generator=g)
    w = torch.randn(n, device=DEV, generator=g) / n
    if form == "moments":
        w = (torch.rand(n, device=DEV, generator=g) < 0.3).float()
    return X, w, mu, sg


def _check_grad(form, got, X, w, mu, sg):
    ref_m, ref_s, tol_m, tol_s = grad_ref(form, X, w, mu, sg, 0.5, 2.0)
    torch.testing.assert_close(got[0].double(), ref_m, rtol=1e-4, atol=tol_m)
    torch.testing.assert_close(got[1].double(), ref_s, rtol=1e-4, atol=tol_s)


# LDG with VEC = 4 and VEC = 1, TMA (D = 512 is the smallest TMA width, D = 1028 leaves a last column tile 4 columns wide)
GRAD_SHAPES = [(20000, 64), (4096, 1030), (8192, 1024), (9000, 1536), (8192, 512), (8192, 1028)]


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("n,D", GRAD_SHAPES)
def test_grad_ignores_padding_and_rows_past_the_end(form, n, D):
    X, w, mu, sg = _grad_data(n, D, n + D, form)
    for pad in (1, 4):  # pad 1: the scalar LDG kernel; pad 4: VEC = 4 / TMA where the shape allows
        runs = [ops.grad(FORMS[form], embed(X, pad, 2, fill), w, mu, sg, 0.5, 2.0) for fill in FILLS]
        _check_grad(form, runs[0], X, w, mu, sg)
        for fill, got in zip(FILLS[1:], runs[1:]):
            assert torch.equal(got[0], runs[0][0]) and torch.equal(got[1], runs[0][1]), f"pad {pad}, fill {fill}"


@pytest.mark.parametrize("form", ["separable", "symmetric", "exp"])
@pytest.mark.parametrize("split", [0, -1])
def test_grad_hybrid_ignores_padding(form, split):
    n, D = 8192, 1024
    g = gen(5)
    mu = torch.randn(D, device=DEV, generator=g)
    sg = torch.rand(D, device=DEV, generator=g) + 0.3
    w = torch.randn(n, device=DEV, generator=g) / n
    sym = form == "symmetric"
    kw = dict(seed=11, stream_id=3, row0=0, scale_mu=0.5, scale_sigma=2.0, split=split)
    for pad in (4, 1, 2, 3):  # pad 4: the TMA / hybrid kernel; pads 1 - 3: the LDG kernel
        runs = []
        for fill in FILLS:
            X = embed(torch.zeros(n, D, device=DEV), pad, 2, fill)
            ops.sample_eval(ops.OBJ_NONE, X, mu, sg, n_rows=n, symmetric=sym, seed=11, stream_id=3)
            runs.append(ops.grad_hybrid(FORMS[form], X, w, mu, sg, **kw))
            if fill == 0.0:
                read = ops.grad(FORMS[form], X, w, mu, sg, 0.5, 2.0)
                assert torch.equal(runs[0][0], read[0]) and torch.equal(runs[0][1], read[1])
                _check_grad(form, runs[0], X, w, mu, sg)
        for fill, got in zip(FILLS[1:], runs[1:]):
            assert torch.equal(got[0], runs[0][0]) and torch.equal(got[1], runs[0][1]), f"pad {pad}, fill {fill}"


# ------------------------------------------------------------------------------------------------ zero-weight rows
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("n_units", [4095, 4096])
@pytest.mark.parametrize("D", [508, 512])
def test_grad_skips_non_finite_rows_whose_weights_are_zero(form, n_units, D, monkeypatch):
    """Rows whose weights are zero (both weights of a direction in the symmetric form) take no part in the gradient, whatever
    they hold -- on both sides of the TMA threshold (n_units >= 4096, D >= 512 with D % 4 == 0)."""
    sym = form == "symmetric"
    n = 2 * n_units if sym else n_units
    X, w, mu, sg = _grad_data(n, D, n_units + D, form)
    units = torch.arange(0, n_units, 7, device=DEV)
    rows = torch.cat([2 * units, 2 * units + 1]) if sym else units
    w[rows] = 0.0
    clean = ops.grad(FORMS[form], X, w, mu, sg, 0.5, 2.0)
    _check_grad(form, clean, X, w, mu, sg)
    for v in POISONS:
        Xp = X.clone()
        Xp[rows] = v
        got = ops.grad(FORMS[form], Xp, w, mu, sg, 0.5, 2.0)
        assert torch.equal(got[0], clean[0]) and torch.equal(got[1], clean[1]), f"zero-weight rows = {v}"
    # the other kernel (LDG when the default is TMA) gives the same answer to fp32 summation order, and also ignores them
    monkeypatch.setenv("EVOK_GRAD_TMA", "0")
    ldg = ops.grad(FORMS[form], Xp, w, mu, sg, 0.5, 2.0)
    monkeypatch.delenv("EVOK_GRAD_TMA")
    _check_grad(form, ldg, X, w, mu, sg)


@pytest.mark.parametrize("form", ["separable", "symmetric", "exp"])
@pytest.mark.parametrize("n_units", [4095, 4096])
@pytest.mark.parametrize("D", [508, 512])
def test_grad_hybrid_skips_non_finite_rows_whose_weights_are_zero(form, n_units, D):
    sym = form == "symmetric"
    n = 2 * n_units if sym else n_units
    g = gen(n + D)
    mu = torch.randn(D, device=DEV, generator=g)
    sg = torch.rand(D, device=DEV, generator=g) + 0.3
    w = torch.randn(n, device=DEV, generator=g) / n
    X = torch.empty(n, D, device=DEV)
    ops.sample_eval(ops.OBJ_NONE, X, mu, sg, n_rows=n, symmetric=sym, seed=21, stream_id=4)
    units = torch.arange(3, n_units, 5, device=DEV)
    rows = torch.cat([2 * units, 2 * units + 1]) if sym else units
    w[rows] = 0.0
    for split in (0, -1, 16):
        kw = dict(seed=21, stream_id=4, row0=0, scale_mu=0.5, scale_sigma=2.0, split=split)
        clean = ops.grad_hybrid(FORMS[form], X, w, mu, sg, **kw)
        _check_grad(form, clean, X, w, mu, sg)
        for v in POISONS:
            Xp = X.clone()
            Xp[rows] = v
            got = ops.grad_hybrid(FORMS[form], Xp, w, mu, sg, **kw)
            assert torch.equal(got[0], clean[0]) and torch.equal(got[1], clean[1]), f"split {split}, zero-weight rows = {v}"


# ------------------------------------------------------------------------------------------------ K6 / K7 matrix kernels
# (M, N, K): K % 4 != 0, and shapes where plan_gemm splits K (few output tiles, long K)
GEMM_SHAPES = [(129, 257, 40), (100, 70, 37), (300, 513, 1000), (129, 130, 999), (2048, 1024, 36)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("pad", [1, 2, 3, 4])  # pad 4: TMA straight from the operands; pads 1 - 3: the pre-split copies
def test_gemm_nt_ignores_padding_and_rows_past_the_end(M, N, K, pad):
    g = gen(M + N + K + pad)
    A = torch.randn(M, K, device=DEV, generator=g)
    B = torch.randn(N, K, device=DEV, generator=g)
    ref = A.double() @ B.double().T
    runs = []
    for fill in FILLS:
        out = embed(torch.zeros(M, N, device=DEV), pad, 3)
        ops.gemm_nt(embed(A, pad, 3, fill), embed(B, pad, 3, fill), out)
        assert_untouched(out, pad, 3)
        runs.append(out.clone())
    assert rel_err(runs[0], ref) < 3e-6
    for fill, got in zip(FILLS[1:], runs[1:]):
        assert torch.equal(got, runs[0]), f"fill {fill}"


@pytest.mark.parametrize("n,d", [(12, 6), (300, 130), (5000, 256), (37, 20), (4096, 1024)])
@pytest.mark.parametrize("pad", [1, 4])
def test_weighted_syrk_update_ignores_padding(n, d, pad):
    g = gen(n + d + pad)
    Y = torch.randn(n, d, device=DEV, generator=g)
    w = torch.randn(n, device=DEV, generator=g) / n
    Cm = torch.randn(d, d, device=DEV, generator=g)
    u = torch.randn(d, device=DEV, generator=g)
    k = torch.tensor([0.7, 0.9, 0.05], device=DEV)
    ref = 0.7 * (Y.double().T * w.double()) @ Y.double() + 0.9 * Cm.double() + 0.05 * torch.outer(u.double(), u.double())
    runs = []
    for fill in FILLS:
        out = embed(torch.zeros(d, d, device=DEV), pad, 2)
        ops.weighted_syrk_update(embed(Y, pad, 2, fill), w, k, embed(Cm, pad, 2, fill), u=u, out=out)
        assert_untouched(out, pad, 2)
        runs.append(out.clone())
    assert rel_err(runs[0], ref) < 3e-6
    for fill, got in zip(FILLS[1:], runs[1:]):
        assert torch.equal(got, runs[0]), f"fill {fill}"


@pytest.mark.parametrize("n", [5, 64, 65, 130, 257])
def test_cholesky_reads_only_the_lower_triangle_inside_the_matrix(n):
    g = gen(n)
    B = torch.randn(n, n, device=DEV, generator=g)
    A = (B @ B.T / n + torch.eye(n, device=DEV) * (0.5 + torch.rand(n, device=DEV, generator=g))).contiguous()
    ref = torch.linalg.cholesky(A.double())
    upper = torch.triu(torch.ones(n, n, dtype=torch.bool, device=DEV), 1)
    runs = []
    for fill in FILLS:
        for pad in (1, 4):
            src = embed(A, pad, 2, fill)
            src[upper] = fill  # strictly above the diagonal
            out = embed(torch.zeros(n, n, device=DEV), pad + 3, 2)
            ops.cholesky(src, out=out)
            assert_untouched(out, pad + 3, 2)
            runs.append(out.clone())
    assert float((runs[0].double() - ref).abs().max()) <= 2e-5 * float(ref.abs().max())
    assert float(runs[0][upper].abs().max() if n > 1 else 0.0) == 0.0
    for got in runs[1:]:
        assert torch.equal(got, runs[0])


@pytest.mark.parametrize("rows,cols", [(67, 64), (67, 37), (300, 130)])
def test_transpose_scale_and_cmaes_row_weights_ignore_padding(rows, cols):
    g = gen(rows + cols)
    X = torch.randn(rows, cols, device=DEV, generator=g)
    w = torch.randn(rows, device=DEV, generator=g)
    assigned = torch.randn(rows, device=DEV, generator=g)
    ref_t = (X.double() * w.double()[:, None]).T
    ref_act = torch.where(assigned > 0, assigned.double(), cols * assigned.double() / (X.double() ** 2).sum(1))
    for pad in (1, 2, 3, 4):
        t_runs, w_runs = [], []
        for fill in FILLS:
            Xv = embed(X, pad, 2, fill)
            t_runs.append(ops.transpose_scale(Xv, w))
            w_pos, w_act = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
            ops.cmaes_row_weights(assigned, Xv, True, w_pos, w_act)
            w_runs.append((w_pos, w_act))
        torch.testing.assert_close(t_runs[0].double(), ref_t, rtol=1e-6, atol=1e-7)
        assert torch.equal(w_runs[0][0], torch.clamp(assigned, min=0.0))
        torch.testing.assert_close(w_runs[0][1].double(), ref_act, rtol=1e-5, atol=1e-7)
        for fill, t, (wp, wa) in zip(FILLS[1:], t_runs[1:], w_runs[1:]):
            assert torch.equal(t, t_runs[0]) and torch.equal(wp, w_runs[0][0]) and torch.equal(wa, w_runs[0][1]), f"pad {pad}, fill {fill}"


# ------------------------------------------------------------------------------------------------ workspace contents
def _poison_workspaces(store: dict, byte: int) -> None:
    for buf in store.values():
        buf.fill_(byte)


def _as_tuple(r):
    return tuple(r) if isinstance(r, (tuple, list)) else (r,)


def _assert_same(a, b, what):
    for x, y in zip(_as_tuple(a), _as_tuple(b)):
        assert torch.equal(x, y), what


def _check_workspace_independence(call, large=None):
    """`call()` returns fresh output tensors.  Its result must not depend on what its workspaces held before: after the shared
    buffers are filled with 0xFF or 0x7F bytes (NaN / a huge float), and after a `large` call left its own data in them, it
    equals a run on private, poisoned, freshly allocated buffers."""
    ref = call()
    for byte in (0xFF, 0x7F):
        _poison_workspaces(nat._workspaces, byte)
        _assert_same(call(), ref, f"workspaces filled with {byte:#x}")
    if large is not None:
        large()
        got = call()
        with nat.private_workspaces() as store:
            call()
            _poison_workspaces(store, 0xFF)
            fresh = call()
        _assert_same(got, fresh, "after a larger call")
        _assert_same(got, ref, "after a larger call (shared buffers)")


RANK_METHODS = ("centered", "linear", "nes", "normalized", "raw")


@pytest.mark.parametrize("n", [1000, 8192, 20000, 524288, 524289, 700000])  # counting path (n <= 8192), self-scanning (n <= 524288) and three-kernel radix sort
def test_ranking_does_not_depend_on_workspace_contents(n):
    g = gen(n)
    f = torch.round(torch.randn(n, device=DEV, generator=g) * 20) / 20  # ties
    big = torch.randn(2 * n + 5000, device=DEV, generator=g)
    table = torch.randn(n, device=DEV, generator=g)

    for method in RANK_METHODS:
        for hib in (False, True):
            def call(method=method, hib=hib):
                perm = torch.empty(n, dtype=torch.int64, device=DEV)
                return ops.rank(f, method, hib, perm=perm), perm

            _check_workspace_independence(call, lambda: ops.rank(big, "centered", True))
    _check_workspace_independence(lambda: ops.argsort(f, True), lambda: ops.argsort(big, True))
    _check_workspace_independence(lambda: ops.rank_table(f, False, table), lambda: ops.argsort(big, False))
    w = ops.rank(f, "raw", True)
    _check_workspace_independence(lambda: ops.elite_mask(w, max(1, n // 4)), lambda: ops.argsort(big, True))
    if n <= 20000:
        fb = torch.round(torch.randn(3, n, device=DEV, generator=g) * 20) / 20
        for method in RANK_METHODS:
            _check_workspace_independence(lambda method=method: ops.rank_batched(fb, method, False),
                                          lambda: ops.rank_batched(torch.randn(5, 2 * n, device=DEV), "nes", True))
        wb = ops.rank_batched(fb, "raw", True)
        _check_workspace_independence(lambda: ops.elite_mask_batched(wb, max(1, n // 4)), lambda: ops.argsort(big, True))


@pytest.mark.parametrize("form", list(FORMS))
def test_gradients_do_not_depend_on_workspace_contents(form):
    fid = FORMS[form]
    sym = form == "symmetric"
    big_X, big_w, big_mu, big_sg = _grad_data(20000, 3000, 1, form)

    def large():
        ops.grad(fid, big_X, big_w, big_mu, big_sg, 1.0, 1.0)

    for n, D in ((2000, 100), (8192, 1024), (4096, 1030)):
        X, w, mu, sg = _grad_data(n, D, n + D, form)
        _check_workspace_independence(lambda: ops.grad(fid, X, w, mu, sg, 0.5, 2.0), large)
        _check_workspace_independence(
            lambda: ops.grad_regen(fid, w, mu, sg, seed=3, stream_id=2, row0=0, scale_mu=0.5, scale_sigma=2.0), large)
        if form != "moments" and D % 4 == 0:
            Xs = torch.empty(n, D, device=DEV)
            ops.sample_eval(ops.OBJ_NONE, Xs, mu, sg, n_rows=n, symmetric=sym, seed=3, stream_id=2)
            _check_workspace_independence(
                lambda: ops.grad_hybrid(fid, Xs, w, mu, sg, seed=3, stream_id=2, row0=0, scale_mu=0.5, scale_sigma=2.0), large)
    Xb = torch.randn(3, 1000, 100, device=DEV, generator=gen(9))
    wb = torch.randn(3, 1000, device=DEV, generator=gen(10)) / 1000
    mub, sgb = torch.zeros(3, 100, device=DEV), torch.ones(3, 100, device=DEV)
    _check_workspace_independence(lambda: ops.grad_batched(fid, Xb, wb, mub, sgb, 0.5, 2.0),
                                  lambda: ops.grad_batched(fid, torch.randn(4, 4000, 300, device=DEV), torch.randn(4, 4000, device=DEV),
                                                           torch.zeros(300, device=DEV), torch.ones(300, device=DEV), 1.0, 1.0))


def test_matrix_kernels_do_not_depend_on_workspace_contents():
    g = gen(2)
    big_A, big_B = torch.randn(600, 3000, device=DEV, generator=g), torch.randn(700, 3000, device=DEV, generator=g)

    def large():
        ops.gemm_nt(big_A, big_B)
        ops.gemm_nt(big_A[:, :2999], big_B[:, :2999])  # the pre-split copies
        ops.weighted_syrk_update(big_A.T.contiguous(), torch.randn(3000, device=DEV), torch.ones(3, device=DEV), torch.randn(600, 600, device=DEV))

    for M, N, K in ((129, 130, 999), (300, 513, 1000), (2048, 1024, 36), (100, 70, 37)):
        A = torch.randn(M, K, device=DEV, generator=g)
        B = torch.randn(N, K, device=DEV, generator=g)
        _check_workspace_independence(lambda: ops.gemm_nt(A, B), large)
        _check_workspace_independence(lambda: ops.gemm_nt(embed(A, 1), embed(B, 3)), large)
    for n, d in ((300, 130), (37, 20), (5000, 256)):
        Y = torch.randn(n, d, device=DEV, generator=g)
        w = torch.randn(n, device=DEV, generator=g) / n
        Cm = torch.randn(d, d, device=DEV, generator=g)
        k = torch.tensor([0.7, 0.9, 0.05], device=DEV)
        _check_workspace_independence(lambda: ops.weighted_syrk_update(Y, w, k, Cm), large)
    big_S = torch.randn(1000, 1000, device=DEV, generator=g)
    big_S = big_S @ big_S.T / 1000 + torch.eye(1000, device=DEV)
    for n in (5, 65, 257):
        B = torch.randn(n, n, device=DEV, generator=g)
        S = (B @ B.T / n + torch.eye(n, device=DEV)).contiguous()
        _check_workspace_independence(lambda: ops.cholesky(S), lambda: ops.cholesky(big_S))


def test_policy_forward_does_not_depend_on_workspace_contents():
    dims, acts = (376, 256, 17), ("tanh", "none")
    g = gen(4)
    P = torch.randn(40, mlp_length(dims), device=DEV, generator=g) * 0.1
    X = torch.randn(40, dims[0], device=DEV, generator=g)
    active = torch.rand(40, device=DEV, generator=g) < 0.6
    big_P = torch.randn(300, mlp_length(dims), device=DEV, generator=g) * 0.1
    big_X = torch.randn(300, dims[0], device=DEV, generator=g)
    # the dynamic ticket of the masked forward lives in the workspace and is zeroed by every call
    _check_workspace_independence(lambda: ops.mlp_forward(P, X, dims, acts, active=active),
                                  lambda: ops.mlp_forward(big_P, big_X, dims, acts, active=torch.ones(300, dtype=torch.bool, device=DEV)))
    x = torch.randn(70, dims[0], device=DEV, generator=g)
    _check_workspace_independence(lambda: ops.mlp_forward_shared(P, x, dims, acts),
                                  lambda: ops.mlp_forward_shared(big_P, torch.randn(256, dims[0], device=DEV), dims, acts))
