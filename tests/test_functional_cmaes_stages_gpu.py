"""Functional CMA-ES on the kernels, stage by stage and generation by generation.

Stages: rank_table_batched, cmaes_row_weights_batched, cmaes_vector_update_batched, evok_transpose_pair_batched and the forms of
gemm_nt_affine_batched / gemm_nt_batched the sampling and SYRK tests leave out.  Every stage writes into buffers with a NaN canary
after the last item that must survive; every item is compared with the single call on that item's own views, bit for bit (the
header's promise), and with float64 under the bounds of test_cmaes_fused.py / test_matrix_kernels.py.  Item counts go up to
70000, where every stage runs as two item chunks: items 0, 65534, 65535, 65536 and the last are probed against the single call.

Whole generations: named cases stepped with cmaes_ask / cmaes_tell, every generation of every item against the float64 oracle
run from the state before it on the tell's own z and fitnesses (`oracle.functional_cmaes_oracle.tell_bound`), each case asserting
the regime it exists for, and a mutation test proving that the bound rejects plausible wrong algorithms.  The ask: x = m +
sigma z A^T over the Philox z of each item."""

import math

import numpy as np
import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import ops
from evotorch_b200.algorithms.cmaes import cmaes_hyperparameters
from evotorch_b200.algorithms.functional import cmaes, cmaes_ask, cmaes_tell, funccmaes
from oracle import es_oracle as O
from oracle import functional_cmaes_oracle as FO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
EPS = 2.0 ** -24
C_ROUND = 4.0  # the rounding constant of test_cmaes_fused.py
BIG = 70000
PROBES = (0, 65534, 65535, 65536, BIG - 1)
_WORST = {}


def _record(name, r):
    _WORST[name] = max(_WORST.get(name, 0.0), r)
    print(f"{name}: worst |err| / bound {r:.3g}")


def ratio(err, bound):
    r = err / bound.clamp_min(1e-300)
    r = torch.where(torch.isfinite(err), r, torch.full_like(r, math.inf))
    return float(r.max()) if r.numel() else 0.0


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def canary(shape, extra=1):
    """A flat NaN buffer for `shape` plus `extra` trailing floats; returns (view of `shape`, the buffer)."""
    n = math.prod(shape)
    buf = torch.full((n + extra,), float("nan"), device=DEV)
    return buf[:n].view(shape), buf


# ------------------------------------------------------------------------------------------------ rank_table_batched
def _keys(g, items, n):
    """Fitnesses with ties inside and across items, +-0, +-inf and NaN."""
    k = torch.randint(-3, 4, (items, n), generator=g).float()
    special = torch.tensor([0.0, -0.0, math.inf, -math.inf, math.nan])
    mask = torch.rand(items, n, generator=g) < 0.3
    k[mask] = special[torch.randint(0, 5, (int(mask.sum()),), generator=g)]
    if items > 1:
        k[1] = k[0]
    return k


def _table(n):
    """The CMA-ES weight table of popsize n (positive head, negative active tail); one value for n = 1."""
    if n == 1:
        return torch.tensor([0.7])
    return cmaes_hyperparameters(4, n, dtype=torch.float32, device="cpu", active=True).weights.float()


RANK_CASES = [(n, b) for n in (1, 2, 7, 1024, 1025, 8192) for b in (1, 5)] + [(n, b) for n in (8193, 20000) for b in (1, 3)]


@pytest.mark.parametrize("n,items", RANK_CASES + [(2, BIG)])
@pytest.mark.parametrize("descending", [False, True])
def test_rank_table_batched(n, items, descending):
    """Exactly the stable reference and, per item, exactly rank_table on that item's keys (above 8192 the per-item radix loop)."""
    g = torch.Generator().manual_seed(n * 7 + items + descending)
    keys = _keys(g, items, n)
    table = _table(n)
    ref = torch.from_numpy(FO.stable_rank_table(keys.numpy(), descending, table.numpy()))
    kd, td = keys.to(DEV), table.to(DEV)
    out, buf = canary((items, n))
    ops.rank_table_batched(kd, descending, td, out=out)
    assert torch.isnan(buf[-1])
    assert same_bits(out.cpu(), ref)
    for b in (range(items) if items <= 5 else PROBES):
        assert same_bits(out[b], ops.rank_table(kd[b].contiguous(), descending, td)), b


# ------------------------------------------------------------------------------------------------ cmaes_row_weights_batched
@pytest.mark.parametrize("n", [1, 7, 8, 9, 4097])
@pytest.mark.parametrize("D", [1, 3, 4, 37, 64, 1025])
@pytest.mark.parametrize("active", [False, True])
def test_row_weights_batched(n, D, active):
    """w_pos = max(a, 0), w_act = a > 0 ? a : D a / ||z||^2 (a without `active`).  Z's item stride is n D + 2 floats, so the
    float4 path (D % 4 == 0) and the scalar path alternate from item to item: each item must get the single call's bits on its
    own view.  Weights positive, +0, -0 and negative; item 0's first row is zero (-inf / NaN where it is reweighted)."""
    items = 4
    g = torch.Generator().manual_seed(n * 11 + D + active)
    stride = n * D + 2
    store = torch.randn(items * stride + 4, generator=g)
    store[:D] = 0.0
    Z = store.to(DEV).as_strided((items, n, D), (stride, D, 1))
    a = torch.randn(items, n, generator=g)
    kind = torch.arange(items * n).view(items, n) % 5
    a = torch.where(kind == 1, torch.zeros_like(a), a)
    a = torch.where(kind == 2, torch.full_like(a, -0.0), a)
    a = torch.where(kind == 3, -a.abs(), a)
    a[0, 0] = -0.5 if n > 1 else -0.0
    a = a.to(DEV)
    w_pos, buf_p = canary((items, n))
    w_act, buf_a = canary((items, n))
    ops.cmaes_row_weights_batched(a, Z, active, w_pos, w_act)
    assert torch.isnan(buf_p[-1]) and torch.isnan(buf_a[-1])
    for b in range(items):
        sp, sa = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        ops.cmaes_row_weights(a[b].contiguous(), Z[b], active, sp, sa)
        assert same_bits(w_pos[b], sp) and same_bits(w_act[b], sa), b
    assert torch.equal(w_pos, torch.clamp_min(a, 0.0))
    z64 = Z.double()
    zn2 = (z64 * z64).sum(-1)
    ref = torch.where(a > 0, a.double(), D * a.double() / zn2) if active else a.double()
    # the zero row: the kernel, its single call (above) and the torch path agree on -inf / NaN
    torch_w = torch.where(a > 0, a, D * a / (Z * Z).sum(-1)) if active else a
    finite = torch.isfinite(ref)
    assert torch.equal(torch.isnan(w_act), torch.isnan(torch_w)) and torch.equal(w_act[~finite & ~torch.isnan(ref)], torch_w[~finite & ~torch.isnan(ref)])
    if active:
        assert not bool(finite[0, 0])
    r = ratio((w_act.double() - ref).abs()[finite], (C_ROUND * EPS * D * ref.abs() + 1e-38)[finite])
    _record("row_weights/w_act", r)
    assert r <= 1.0


def test_row_weights_batched_takes_any_stride_of_a_unit_dimension():
    """torch leaves the stride of a size-1 dimension arbitrary, even in a contiguous tensor: the z of a D = 1 tell is (items, n, 1)
    with strides (n, 1, n).  Such a Z is accepted and read as the same memory."""
    Z = torch.randn(3 * 4, device=DEV).as_strided((3, 4, 1), (4, 1, 4))
    a = torch.randn(3, 4, device=DEV) - 0.5
    w_pos, w_act = torch.empty(3, 4, device=DEV), torch.empty(3, 4, device=DEV)
    ops.cmaes_row_weights_batched(a, Z, True, w_pos, w_act)
    Zc = Z.reshape(3, 4).clone().view(3, 4, 1)
    p2, a2 = torch.empty(3, 4, device=DEV), torch.empty(3, 4, device=DEV)
    ops.cmaes_row_weights_batched(a, Zc, True, p2, a2)
    assert same_bits(w_pos, p2) and same_bits(w_act, a2)


def test_row_weights_batched_across_item_chunks():
    g = torch.Generator().manual_seed(1)
    n, D = 7, 4
    stride = n * D + 2
    Z = torch.randn(BIG * stride, generator=g).to(DEV).as_strided((BIG, n, D), (stride, D, 1))
    a = (torch.randn(BIG, n, generator=g) - 0.3).to(DEV)
    w_pos, buf_p = canary((BIG, n))
    w_act, buf_a = canary((BIG, n))
    ops.cmaes_row_weights_batched(a, Z, True, w_pos, w_act)
    assert torch.isnan(buf_p[-1]) and torch.isnan(buf_a[-1])
    for b in PROBES:
        sp, sa = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        ops.cmaes_row_weights(a[b].contiguous(), Z[b], True, sp, sa)
        assert same_bits(w_pos[b], sp) and same_bits(w_act[b], sa), b
    z64 = Z.double()
    ref = torch.where(a > 0, a.double(), D * a.double() / (z64 * z64).sum(-1))
    assert torch.equal(w_pos, torch.clamp_min(a, 0.0))
    assert ratio((w_act.double() - ref).abs(), C_ROUND * EPS * D * ref.abs() + 1e-38) <= 1.0


# ------------------------------------------------------------------------------------------------ cmaes_vector_update_batched
def _consts(st):
    return (st.c_m, st.c_sigma, st.damp_sigma, st.c_c, st.c_1, st.c_mu, st.variance_discount_sigma, st.variance_discount_c,
            float(st.unbiased_expectation), float(np.sum(st.weights, dtype=np.float32)))


def _vector_case(D, csa_squared, steps, items, seed):
    """Per item a state whose ||p_sigma'||^2 lands 30 % below (even items) or above (odd items) the h_sig threshold
    (the construction of test_cmaes_fused.test_vector_update_matches_the_oracle_vector_step)."""
    rng = np.random.default_rng(seed)
    n = max(4 + int(np.floor(3 * np.log(D))), 6)
    st = O.CMAESState(D, n, 0.7, np.zeros(D), csa_squared=bool(csa_squared))
    decay = 1 - (1 - st.c_sigma) ** (2 * steps + 1)
    rhs = 1 + 4.0 / (D + 1)
    p_sigma0 = rng.standard_normal((items, D))
    local = rng.standard_normal((items, D))
    v = (1 - st.c_sigma) * p_sigma0 + st.variance_discount_sigma * local
    h_target = np.where(np.arange(items) % 2 == 0, 1.0, 0.0)
    target = (rhs * np.where(h_target == 1.0, 0.7, 1.3) + 1) * D * decay
    s = np.sqrt(target / (v * v).sum(-1))[:, None]
    f32 = np.float32
    state = dict(m=rng.uniform(-2, 2, (items, D)).astype(f32), p_sigma=(p_sigma0 * s).astype(f32), p_c=(rng.standard_normal((items, D)) * 0.2).astype(f32),
                 sigma=rng.uniform(0.3, 1.5, items).astype(f32), local=(local * s).astype(f32),
                 shaped=(rng.standard_normal((items, D)) * 0.5).astype(f32))
    return st, state, h_target


def _vector_check(st, s0, b, steps, got, h_expect):
    """One item against O.cmaes_vector_step and O.cmaes_k under the bounds of test_cmaes_fused; h_sig exactly."""
    o = O.CMAESState(st.d, st.popsize, float(s0["sigma"][b]), s0["m"][b], csa_squared=st.csa_squared)
    o.c_m, o.c_sigma, o.damp_sigma, o.c_c, o.c_1, o.c_mu = st.c_m, st.c_sigma, st.damp_sigma, st.c_c, st.c_1, st.c_mu
    o.p_sigma, o.p_c, o.sigma, o.steps = s0["p_sigma"][b].copy(), s0["p_c"][b].copy(), np.float32(s0["sigma"][b]), steps
    local, shaped = s0["local"][b].astype(np.float64), s0["shaped"][b].astype(np.float64)
    h = O.cmaes_vector_step(o, local, shaped)
    _, margin = O.cmaes_h_sig(o, float(np.linalg.norm(o.p_sigma.astype(np.float64))))
    assert h == h_expect and margin > 0.1
    tol = C_ROUND * EPS
    sig0 = float(s0["sigma"][b])
    pnorm = float(np.linalg.norm(o.p_sigma.astype(np.float64)))
    mag_expo = pnorm**2 / st.d if st.csa_squared else pnorm / o.unbiased_expectation
    k_ref = O.cmaes_k(o, h)
    c1a, _ = O.cmaes_covariance_coefficients(o, h)
    wsum = float(np.sum(o.weights, dtype=np.float32))
    k_mag = np.array([abs(o.c_mu), 1 + c1a + abs(o.c_mu * wsum), 3 * abs(k_ref[2])])
    checks = (("m", got["m"][b], o.m, tol * (np.abs(s0["m"][b]) + abs(o.c_m * sig0) * np.abs(shaped))),
              ("p_sigma", got["p_sigma"][b], o.p_sigma, tol * (abs(1 - o.c_sigma) * np.abs(s0["p_sigma"][b]) + o.variance_discount_sigma * np.abs(local))),
              ("p_c", got["p_c"][b], o.p_c, tol * (abs(1 - o.c_c) * np.abs(s0["p_c"][b]) + h * o.variance_discount_c * np.abs(shaped))),
              ("sigma", got["sigma"][b], float(o.sigma), tol * float(o.sigma) * (4 + (o.c_sigma / o.damp_sigma) * 4 * mag_expo)),
              ("k", got["k"][b], np.array(k_ref), tol * k_mag))
    worst = 0.0
    for name, g_, r_, bound in checks:
        err = np.abs(np.asarray(g_, np.float64) - np.asarray(r_, np.float64))
        q = float(np.max(np.where(np.isfinite(err), err / (np.asarray(bound) + 1e-30), np.inf)))
        assert q <= 1.0, (b, name, q)
        worst = max(worst, q)
    # h_sig exactly: p_c of the other branch lies far outside the bound.  (k_out does not show h_sig in general: k_out[2] =
    # c1a c_1 / c1a is c_1 on both branches, and with active weights c_mu sum(w) ~ -c_1 leaves k_out[1] ~ 1 on both.)
    pc_other = (1 - o.c_c) * s0["p_c"][b].astype(np.float64) + (1.0 - h) * o.variance_discount_c * shaped
    bound_pc = checks[2][3] + 1e-30
    assert np.max(np.abs(got["p_c"][b] - pc_other) / bound_pc) > 1e3, b
    return worst


def _run_vector_update(D, csa_squared, steps, items, seed):
    st, s0, h_target = _vector_case(D, csa_squared, steps, items, seed)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in s0.items()}
    bufs = {}
    for name in ("m", "p_sigma", "p_c", "sigma"):
        view, bufs[name] = canary(tuple(t[name].shape))
        view.copy_(t[name])
        t[name] = view
    t["k"], bufs["k"] = canary((items, 3))
    single = {name: t[name].clone() for name in ("m", "p_sigma", "p_c", "sigma")}
    ops.cmaes_vector_update_batched(t["local"], t["shaped"], t["m"], t["p_sigma"], t["p_c"], t["sigma"], _consts(st), bool(csa_squared), t["k"], steps=steps)
    for name, buf in bufs.items():
        assert torch.isnan(buf[-1]), name
    probes = range(items) if items <= 8 else PROBES
    for b in probes:
        m, ps, pc = (single[n][b].clone() for n in ("m", "p_sigma", "p_c"))
        sg = single["sigma"][b:b + 1].clone()
        k = torch.empty(3, device=DEV)
        ops.cmaes_vector_update(t["local"][b].contiguous(), t["shaped"][b].contiguous(), m, ps, pc, sg, _consts(st), bool(csa_squared), k, steps=steps)
        for got, want in ((t["m"][b], m), (t["p_sigma"][b], ps), (t["p_c"][b], pc), (t["sigma"][b:b + 1], sg), (t["k"][b], k)):
            assert same_bits(got, want), b
    got = {n: t[n].cpu().numpy() for n in ("m", "p_sigma", "p_c", "sigma", "k")}
    check_items = range(items) if items <= 8 else sorted(set(PROBES) | set(range(0, items, 997)))
    worst = max(_vector_check(st, s0, b, steps, got, h_target[b]) for b in check_items)
    return worst, bufs


@pytest.mark.parametrize("D", [1, 2, 31, 1024, 1025, 5000])
@pytest.mark.parametrize("csa_squared", [False, True])
@pytest.mark.parametrize("steps", [0, 3, 10**6])
def test_vector_update_batched(D, csa_squared, steps):
    """Four items in one launch, two landing 30 % below the h_sig threshold and two 30 % above: the branch is taken per item.
    m, p_sigma, p_c, sigma and k_out of each item are the single call's bits and within the oracle's bound; h_sig is exact."""
    worst, _ = _run_vector_update(D, csa_squared, steps, 4, D * 10 + steps % 7 + csa_squared)
    _record("vector_update", worst)


def test_vector_update_batched_across_item_chunks():
    worst, _ = _run_vector_update(2, False, 3, BIG, 5)
    _record("vector_update/70000", worst)


# ------------------------------------------------------------------------------------------------ evok_transpose_pair_batched
def _transpose(items, rows, cols, shared_w, seed):
    g = torch.Generator().manual_seed(seed)
    ldi = cols + 1
    s_in = rows * ldi + 3
    inp = torch.randn(items * s_in + 8, generator=g).to(DEV)
    Y = inp.as_strided((items, rows, cols), (s_in, ldi, 1))
    w = torch.randn(rows if shared_w else items * rows, generator=g).to(DEV)
    ldo = rows + 5
    s_out = cols * ldo + 7
    out_w = torch.full((items * s_out + 16,), float("nan"), device=DEV)
    out_p = torch.full((items * s_out + 16,), float("nan"), device=DEV)
    rc = nat.lib().evok_transpose_pair_batched(inp.data_ptr(), ldi, s_in, rows, cols, w.data_ptr(), 0 if shared_w else rows, out_w.data_ptr(),
                                               out_p.data_ptr(), ldo, s_out, items, nat.stream_of(inp))
    nat.check(rc, "evok_transpose_pair_batched")
    ow = out_w[:items * s_out].view(items, s_out)
    op = out_p[:items * s_out].view(items, s_out)
    W = w.view(1, rows).expand(items, rows) if shared_w else w.view(items, rows)
    want_w = (Y * W[:, :, None]).mT  # fp32 products, as the kernel forms them
    want_p = Y.mT
    got_w = ow[:, :cols * ldo].view(items, cols, ldo)
    got_p = op[:, :cols * ldo].view(items, cols, ldo)
    return dict(got_w=got_w, got_p=got_p, want_w=want_w, want_p=want_p, ow=ow, op=op, out_w=out_w, out_p=out_p, rows=rows, cols=cols, ldo=ldo,
                s_out=s_out, items=items)


def _transpose_asserts(t, check_items):
    rows, cols = t["rows"], t["cols"]
    for b in check_items:
        assert same_bits(t["got_w"][b, :, :rows], t["want_w"][b]), b
        assert same_bits(t["got_p"][b, :, :rows], t["want_p"][b]), b
    # the padding columns between rows and ldo, the gap between items and everything past the last item stay untouched
    assert torch.isnan(t["got_w"][:, :, rows:]).all() and torch.isnan(t["got_p"][:, :, rows:]).all()
    assert torch.isnan(t["ow"][:, cols * t["ldo"]:]).all() and torch.isnan(t["op"][:, cols * t["ldo"]:]).all()
    assert torch.isnan(t["out_w"][t["items"] * t["s_out"]:]).all() and torch.isnan(t["out_p"][t["items"] * t["s_out"]:]).all()


@pytest.mark.parametrize("rows", [1, 31, 33, 300, 8193])
@pytest.mark.parametrize("cols", [1, 33, 130])
@pytest.mark.parametrize("items", [1, 3])
@pytest.mark.parametrize("shared_w", [False, True])
def test_transpose_pair_batched(rows, cols, items, shared_w):
    """out_w = fp32(w Y)^T and out_p = Y^T exactly, with padded input and output item strides and a shared or per-item w."""
    t = _transpose(items, rows, cols, shared_w, rows * 3 + cols + items + shared_w)
    _transpose_asserts(t, range(items))


def test_transpose_pair_batched_across_item_chunks():
    t = _transpose(BIG, 2, 3, False, 9)
    _transpose_asserts(t, PROBES)
    assert same_bits(t["got_w"][:, :, :2], t["want_w"]) and same_bits(t["got_p"][:, :, :2], t["want_p"])


# ------------------------------------------------------------------------------------------------ gemm_nt_affine_batched / gemm_nt_batched
BM = BN = 128
SMS = 132


def one_split(M, N, K):
    """True when gemm_nt's plan for this shape has one K split (the batched plan never splits)."""
    tiles = -(-M // BM) * -(-N // BN)
    return tiles * 2 > SMS or -(-K // FO.BK) < 2


def gemm_nt_affine(A, B, k, out, E=None, u=None):
    """The single call evok_gemm_nt_affine on 2-D views (row-major rows, any pitch)."""
    M, K = A.shape
    N = B.shape[0]
    lib = nat.lib()
    ws = nat.workspace(A.device, lib.evok_gemm_workspace_bytes(M, N, K), "gemm")
    rc = lib.evok_gemm_nt_affine(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), M, N, K, out.data_ptr(), out.stride(0), k.data_ptr(), nat.ptr(E),
                                 0 if E is None else E.stride(0), nat.ptr(u), ws.data_ptr(), ws.numel(), nat.stream_of(A))
    nat.check(rc, "evok_gemm_nt_affine")
    return out


def _operand(g, items, rows, cols, form):
    """aligned (items, rows, cols); unaligned: row pitch cols + 1 and item pitch rows (cols + 1) + 1; shared: (rows, cols)."""
    if form == "shared":
        return torch.randn(rows, cols, generator=g).to(DEV)
    if form == "shared_unaligned":
        flat = torch.randn(rows * (cols + 1) + 2, generator=g).to(DEV)
        return flat.as_strided((rows, cols), (cols + 1, 1), 1)
    if form == "aligned":
        return torch.randn(items, rows, cols, generator=g).to(DEV)
    flat = torch.randn(items * (rows * (cols + 1) + 1) + 8, generator=g).to(DEV)
    return flat.as_strided((items, rows, cols), (rows * (cols + 1) + 1, cols + 1, 1), 1)


AFFINE_FORMS = {
    # name: (A form, B form, k shared, E: "item" / "shared" / None / "out", u: "item" / "shared" / None, coefficients)
    "shared_k": ("aligned", "aligned", True, "item", "item", "random"),
    "shared_E": ("aligned", "aligned", False, "shared", "item", "random"),
    "shared_u": ("aligned", "aligned", False, "item", "shared", "random"),
    "no_E_no_u": ("aligned", "aligned", False, None, None, "random"),
    "no_u": ("unaligned", "aligned", False, "item", None, "random"),
    "in_place": ("aligned", "aligned", False, "out", "item", "random"),
    "in_place_unaligned": ("unaligned", "unaligned", False, "out", "item", "random"),
    "k0_zero": ("aligned", "aligned", False, "item", "item", "k0_zero"),
    "negative": ("aligned", "aligned", False, "item", "item", "negative"),
    "aligned_A_shared_unaligned_B": ("aligned", "shared_unaligned", False, "item", "item", "random"),
}


@pytest.mark.parametrize("form", list(AFFINE_FORMS))
@pytest.mark.parametrize("M,K,items", [(3, 5, 1), (3, 5, 4), (33, 17, 4), (130, 300, 3)])
def test_gemm_nt_affine_batched_forms(form, M, K, items):
    """out_b = k_b0 A_b B_b^T + k_b1 E_b + k_b2 u_b u_b^T with shared k / E / u, without E or u, in place (out is E: the
    out-of-place bits), k0 = 0 and negative coefficients, and a per-item aligned A with a shared unaligned B (both operands
    through the split copies).  Per item the single call's bits where its plan has one split; everywhere the K7 bound."""
    fa, fb, k_shared, e_form, u_form, coef = AFFINE_FORMS[form]
    N = M
    g = torch.Generator().manual_seed(list(AFFINE_FORMS).index(form) * 1000 + M * 10 + K + items)
    A = _operand(g, items, M, K, fa)
    B = _operand(g, items, N, K, fb)
    k = torch.rand(3 if k_shared else items * 3, generator=g) + 0.1
    if coef == "k0_zero":
        k.view(-1, 3)[:, 0] = 0.0
    if coef == "negative":
        k = -k
    k = (k if k_shared else k.view(items, 3)).to(DEV)
    E_src = None if e_form is None else torch.randn(*(() if e_form == "shared" else (items,)), M, N, generator=g).to(DEV)
    u = None if u_form is None else torch.randn(*(() if u_form == "shared" else (items,)), M, generator=g).to(DEV)
    out, buf = canary((items, M, N))
    if e_form == "out":
        out.copy_(E_src)
        E = out
    else:
        E = E_src
    ops.gemm_nt_affine_batched(A, B, k, out, E=E, u=u)
    assert torch.isnan(buf[-1])
    if e_form == "out":  # in place: the bits of the same call out of place
        ref_out = torch.empty(items, M, N, device=DEV)
        ops.gemm_nt_affine_batched(A, B, k, ref_out, E=E_src, u=u)
        assert same_bits(out, ref_out)
    Ai = lambda b: A if A.ndim == 2 else A[b]  # noqa: E731
    Bi = lambda b: B if B.ndim == 2 else B[b]  # noqa: E731
    ki = lambda b: k if k.ndim == 1 else k[b]  # noqa: E731
    Ei = lambda b: None if E_src is None else (E_src if E_src.ndim == 2 else E_src[b])  # noqa: E731
    ui = lambda b: None if u is None else (u if u.ndim == 1 else u[b])  # noqa: E731
    if one_split(M, N, K):
        for b in range(items):
            single = gemm_nt_affine(Ai(b), Bi(b), ki(b).contiguous(), torch.empty(M, N, device=DEV), E=Ei(b), u=ui(b))
            assert same_bits(out[b], single), b
    A64 = (A if A.ndim == 3 else A.expand(items, M, K)).double()
    B64 = (B if B.ndim == 3 else B.expand(items, N, K)).double()
    k64 = (k if k.ndim == 2 else k.expand(items, 3)).double()
    acc = A64 @ B64.mT
    absab = A64.abs() @ B64.abs().mT
    Ed = torch.zeros(items, M, N, dtype=torch.float64, device=DEV) if E_src is None else E_src.double().expand(items, M, N)
    uu = torch.zeros(items, M, N, dtype=torch.float64, device=DEV) if u is None else (u.double()[..., :, None] * u.double()[..., None, :]).expand(items, M, N)
    k0, k1, k2 = (k64[:, i, None, None] for i in range(3))
    ref = k0 * acc + k1 * Ed + k2 * uu
    bound = k0.abs() * FO.gamma(K) * absab + EPS * (k0.abs() * acc.abs() + 2 * k1.abs() * Ed.abs() + 3 * k2.abs() * uu.abs()) + 1e-300
    r = ratio((out.double() - ref).abs(), bound)
    _record("gemm_affine", r)
    assert r <= 1.0


@pytest.mark.parametrize("epilogue", ["alpha_only", "bias_only", "shared_bias", "shared_alpha"])
@pytest.mark.parametrize("M,N,K,items", [(4, 3, 5, 3), (40, 33, 17, 4), (130, 129, 64, 2)])
def test_gemm_nt_batched_second_output(epilogue, M, N, K, items):
    """out2_b = alpha_b out_b + bias_b with only one of alpha / bias, or one shared by the items: per item the bits of gemm_nt with
    the same second output, and out within the K6 bound."""
    g = torch.Generator().manual_seed(M * N + K + items)
    A = torch.randn(items, M, K, generator=g).to(DEV)
    B = torch.randn(items, N, K, generator=g).to(DEV)
    alpha = None if epilogue == "bias_only" else (torch.rand(1 if epilogue == "shared_alpha" else items, generator=g) + 0.5).to(DEV)
    bias = None if epilogue == "alpha_only" else torch.randn(*(() if epilogue == "shared_bias" else (items,)), N, generator=g).to(DEV)
    out, buf1 = canary((items, M, N))
    out2, buf2 = canary((items, M, N))
    ops.gemm_nt_batched(A, B, out, out2=out2, alpha=alpha, bias=bias)
    assert torch.isnan(buf1[-1]) and torch.isnan(buf2[-1])
    for b in range(items):
        y, x = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
        ab = None if alpha is None else (alpha if alpha.numel() == 1 else alpha[b:b + 1])
        bb = None if bias is None else (bias if bias.ndim == 1 else bias[b])
        ops.gemm_nt(A[b], B[b], y, out2=x, alpha=ab, bias=bb)  # out2: the single call never splits K
        assert same_bits(out[b], y) and same_bits(out2[b], x), b
    ref = A.double() @ B.double().mT
    r = ratio((out.double() - ref).abs(), FO.gamma(K) * (A.double().abs() @ B.double().abs().mT) + 1e-300)
    _record("gemm_nt_batched/out", r)
    assert r <= 1.0
    a64 = torch.ones(items, 1, 1, dtype=torch.float64, device=DEV) if alpha is None else alpha.double().expand(items).view(items, 1, 1)
    b64 = torch.zeros(items, 1, N, dtype=torch.float64, device=DEV) if bias is None else bias.double().expand(items, N).view(items, 1, N)
    # out2 = fmaf(alpha, out, bias): one rounding on top of out's own
    want2 = a64 * out.double() + b64
    assert ratio((out2.double() - want2).abs(), EPS * want2.abs() + 1e-300) <= 1.0


def test_gemm_affine_batched_across_item_chunks():
    """70000 items of the covariance-update form (per-item k, E in place, u): probes against the single call, all against float64."""
    g = torch.Generator().manual_seed(12)
    M, K = 3, 5
    A = torch.randn(BIG, M, K, generator=g).to(DEV)
    B = torch.randn(BIG, M, K, generator=g).to(DEV)
    k = (torch.rand(BIG, 3, generator=g) - 0.3).to(DEV)
    u = torch.randn(BIG, M, generator=g).to(DEV)
    out, buf = canary((BIG, M, M))
    out.copy_(torch.randn(BIG, M, M, generator=g).to(DEV))
    E0 = out.clone()
    ops.gemm_nt_affine_batched(A, B, k, out, E=out, u=u)
    assert torch.isnan(buf[-1])
    for b in PROBES:
        assert same_bits(out[b], gemm_nt_affine(A[b], B[b], k[b].contiguous(), torch.empty(M, M, device=DEV), E=E0[b], u=u[b])), b
    k64 = k.double()
    acc = A.double() @ B.double().mT
    uu = u.double()[:, :, None] * u.double()[:, None, :]
    k0, k1, k2 = (k64[:, i, None, None] for i in range(3))
    ref = k0 * acc + k1 * E0.double() + k2 * uu
    bound = k0.abs() * FO.gamma(K) * (A.double().abs() @ B.double().abs().mT) + EPS * (k0.abs() * acc.abs() + 2 * k1.abs() * E0.double().abs()
                                                                                       + 3 * k2.abs() * uu.abs()) + 1e-300
    assert ratio((out.double() - ref).abs(), bound) <= 1.0


# ------------------------------------------------------------------------------------------------ whole generations
def _ellipsoid(x):
    d = x.shape[-1]
    scale = 10.0 ** (3 * torch.arange(d, device=x.device, dtype=x.dtype) / max(d - 1, 1))
    return (scale * x * x).sum(-1)


def _sphere(x):
    return (x * x).sum(-1)


def _mixed_linear(x):
    """Linear (sigma collapses, ||p_sigma|| grows: h_sig = 0) on the even items of a flat batch, sphere around the centre
    (h_sig = 1) on the odd ones."""
    items = x.shape[0]
    lin = x.sum(-1)
    sph = ((x - x.mean(-2, keepdim=True)) ** 2).sum(-1)
    even = (torch.arange(items, device=x.device) % 2 == 0)[:, None]
    return torch.where(even, lin, sph)


def _nonfinite(x):
    f = -_sphere(x)
    r = torch.arange(f.shape[-1], device=x.device)
    f = torch.where(r % 7 == 3, torch.full_like(f, float("nan")), f)
    f = torch.where(r % 11 == 5, torch.full_like(f, float("inf")), f)
    return torch.where(r % 13 == 8, torch.full_like(f, float("-inf")), f)


# name: (batch shape, D, objective, options of cmaes(), generations)
GEN_CASES = {
    "D1": ((3,), 1, _sphere, {}, 10),
    "D2": ((3,), 2, _ellipsoid, {}, 10),
    "D1025": ((2,), 1025, _sphere, {}, 17),
    "radix": ((2,), 129, _sphere, {"popsize": 8193}, 3),
    "h_sig_mixed": ((4,), 10, _mixed_linear, {"stdev_init": 1e-3}, 14),
    "max_active_nonfinite": ((3,), 20, _nonfinite, {"objective_sense": "max", "popsize": 40}, 6),
    "stdev_clamp": ((3,), 10, _ellipsoid, {"stdev_init": 0.3, "stdev_min": 0.29, "stdev_max": 100.0}, 8),
    "csa_squared_passive": ((3,), 12, _ellipsoid, {"active": False, "csa_squared": True}, 8),
    "shape_scalar": ((), 5, _ellipsoid, {}, 6),
    "shape_3x4": ((3, 4), 4, _ellipsoid, {}, 6),
    "items_70000": ((BIG,), 2, _sphere, {}, 2),
}
_GEN_RUNS = {}


def _run_generations(name):
    """Step the case with cmaes_ask / cmaes_tell, checking every generation of every item against the oracle, and measure every
    mutated reference.  Returns what the case reached and, per mutation, the largest error / bound it produced."""
    if name in _GEN_RUNS:
        return _GEN_RUNS[name]
    batch, d, fn, kw, gens = GEN_CASES[name]
    kw = dict(kw)
    torch.manual_seed(len(name) * 31 + d)
    state = cmaes(center_init=torch.randn(*batch, d, device=DEV), stdev_init=kw.pop("stdev_init", 1.0), objective_sense=kw.pop("objective_sense", "min"),
                  **kw)
    B = math.prod(batch)
    check = list(range(B)) if B <= 16 else list(PROBES)
    seen = dict(h=set(), h_mixed=False, min_margin=math.inf, due=set(), clamp=False, worst=0.0)
    caught = {mut: 0.0 for mut in FO.MUTATIONS}
    for gen in range(gens):
        x = cmaes_ask(state)
        f = fn(x.reshape(B, state.popsize, d)).reshape(batch + (state.popsize,))
        new = cmaes_tell(state, x, f)
        fs, fnew = FO.flat_state(state), FO.flat_state(new)
        xf, ff = x.reshape(B, state.popsize, d), f.reshape(B, state.popsize)
        rec = []
        r = max(FO.tell_bound(fs, xf, ff, fnew, items=check, record=rec))
        assert r <= 1.0, (name, gen, r)
        seen["worst"] = max(seen["worst"], r)
        hs = {o["h"] for o in rec}
        seen["h"] |= hs
        seen["h_mixed"] |= len(hs) == 2
        seen["min_margin"] = min(seen["min_margin"], min(o["margin"] for o in rec))
        if state.stdev_min is not None:
            seen["clamp"] |= any(bool(((o["stdevs"] < state.stdev_min) | (o["stdevs"] > state.stdev_max)).any()
                                      and ((o["stdevs"] >= state.stdev_min) & (o["stdevs"] <= state.stdev_max)).any()) for o in rec)
        due = (state.generation + 1) % state.hyperparameters.decompose_C_freq == 0
        seen["due"].add(due)
        if due:  # A refactorised from the new C: within a Cholesky bound of float64
            C64 = fnew.C[check].double()
            L = torch.linalg.cholesky(C64)
            dg = torch.diagonal(C64, dim1=-2, dim2=-1).abs().sqrt()
            bound = C_ROUND * EPS * (state.popsize + d) * dg[:, :, None] * dg[:, None, :] + 1e-30  # test_cmaes_fused's bound of A
            assert ratio((fnew.A[check].double() - L).abs(), bound) <= 1.0, (name, gen)
        else:
            assert torch.equal(fnew.A, fs.A), (name, gen)
        if B > 1000:  # every item against the batched torch path on the CPU in float64, loosely
            cpu = lambda t: t.detach().double().cpu()  # noqa: E731
            s64 = state._replace(center=cpu(state.center), sigma=cpu(state.sigma), C=cpu(state.C), A=cpu(state.A), p_sigma=cpu(state.p_sigma),
                                 p_c=cpu(state.p_c), hyperparameters=state.hyperparameters._replace(weights=cpu(state.hyperparameters.weights)))
            t64 = cmaes_tell(s64, cpu(x), cpu(f))
            for field in ("center", "sigma", "C", "p_sigma", "p_c"):
                a, b = getattr(new, field).double().cpu(), getattr(t64, field)
                assert torch.allclose(a, b, rtol=1e-3, atol=1e-4 * float(b.abs().max())), (name, gen, field)
        for mut in FO.MUTATIONS:
            if caught[mut] <= 1.0:
                caught[mut] = max(caught[mut], max(FO.tell_bound(fs, xf, ff, fnew, mutation=mut, items=check)))
        state = new
    _GEN_RUNS[name] = (seen, caught)
    return _GEN_RUNS[name]


@pytest.mark.parametrize("case", list(GEN_CASES))
def test_generations_match_the_float64_oracle(case):
    """Every generation of every checked item (all items, or the chunk-edge probes of 70000) against the oracle under the
    first-order bound; A bit-identical on generations without a decomposition and refactorised on the others.  Each case
    reaches what it is there for; no generation comes within 1e-4 (relative) of the h_sig threshold."""
    seen, _ = _run_generations(case)
    print(f"{case}: worst |err| / bound {seen['worst']:.3g}, h_sig {sorted(seen['h'])}, min margin {seen['min_margin']:.3g}")
    _record(f"gen/{case}", seen["worst"])
    assert seen["min_margin"] > 1e-4, seen["min_margin"]
    if case == "D1025":
        assert seen["due"] == {True, False}
    if case == "radix":
        assert GEN_CASES[case][3]["popsize"] > 8192
    if case == "h_sig_mixed":
        assert seen["h_mixed"], "h_sig = 0 and h_sig = 1 among the items of one generation"
    if case == "stdev_clamp":
        assert seen["clamp"], "the clamp active on some diagonal entries and not on others"


def test_every_mutated_reference_is_rejected_by_some_case():
    """The bound is tight enough to matter: each mutated reference falls outside it in at least one case."""
    caught = {mut: [] for mut in FO.MUTATIONS}
    for case in GEN_CASES:
        for mut, r in _run_generations(case)[1].items():
            if r > 1.0:
                caught[mut].append(case)
    print("worst error / bound:", {k: round(v, 3) for k, v in sorted(_WORST.items())})
    print("mutations caught by:", caught)
    missed = [mut for mut, cases in caught.items() if not cases]
    assert not missed, f"mutated references inside the bounds of every case: {missed}; caught: {caught}"


# ------------------------------------------------------------------------------------------------ the ask
SEED = 987654321


@pytest.mark.parametrize("case", ["split_D5", "noncontiguous_A", "shape_scalar", "shape_3x4", "items_70000"])
def test_ask_is_the_sampling_product_of_the_philox_z(case, monkeypatch):
    """x = m_b + sigma_b z_b A_b^T over z_b = item b's Philox stream (regenerated with sample_batched), within the K6 bound of
    float64; at 70000 items no two items around the chunk edge share their z."""
    monkeypatch.setattr(funccmaes, "draw_philox_seed", lambda: SEED)
    batch, d = {"split_D5": ((3,), 5), "noncontiguous_A": ((4,), 6), "shape_scalar": ((), 7), "shape_3x4": ((3, 4), 4), "items_70000": ((BIG,), 2)}[case]
    torch.manual_seed(3)
    state = cmaes(center_init=torch.randn(*batch, d, device=DEV), stdev_init=torch.rand(batch, device=DEV) + 0.5, objective_sense="min")
    B = math.prod(batch)
    L = torch.randn(B, d, d, device=DEV).tril() + 2 * torch.eye(d, device=DEV)
    if case == "noncontiguous_A":
        big = torch.randn(2 * B, d, d, device=DEV)
        big[::2] = L
        A = big[::2]
        assert not A.is_contiguous()
    else:
        A = L.reshape(batch + (d, d))
    state = state._replace(A=A)
    x = cmaes_ask(state)
    assert x.shape == batch + (state.popsize, d)
    n = state.popsize
    z = torch.empty(B, n, d, device=DEV)
    zero = torch.zeros(d, device=DEV)
    ops.sample_batched(z, zero, zero + 1.0, symmetric=False, seed=SEED)
    m64, s64, A64 = state.center.reshape(B, d).double(), state.sigma.reshape(B).double(), L.double()
    zA = z.double() @ A64.mT
    ref = m64[:, None, :] + s64[:, None, None] * zA
    mag = m64.abs()[:, None, :] + s64[:, None, None] * (z.double().abs() @ A64.abs().mT)
    bound = s64[:, None, None] * FO.gamma(d) * (z.double().abs() @ A64.abs().mT) + 2 * EPS * mag + 1e-30
    r = ratio((x.reshape(B, n, d).double() - ref).abs(), bound)
    _record(f"ask/{case}", r)
    assert r <= 1.0
    if B == BIG:
        edge = z[65530:65541].reshape(11, -1)
        assert torch.unique(edge, dim=0).shape[0] == 11
        assert not any(torch.equal(z[b], z[b - 65535]) for b in (65535, 65536, BIG - 1))
