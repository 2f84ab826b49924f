"""The dense-matrix kernels K6 / K7 -- the 3xTF32 GEMM (csrc/evok_gemm.cu) and the tile-dataflow Cholesky (csrc/evok_chol.cu) --
element by element against float64, at the shapes, layouts, epilogues and data where such kernels go wrong.

GEMM  C = A B^T  (`ops.gemm_nt`, and `evok_gemm_nt_affine` behind `ops.weighted_syrk_update`).  Per element:

    |C - C64|_ij <= C_ROUND * gamma * (|A||B|^T)_ij  (+ epilogue terms)
    gamma = 3 * 2^-20 + 2^-24 * (K_chunk + splits + 2)

  * 3 * 2^-20: every operand is split as x = hi + lo, hi = x with the 13 low mantissa bits cleared, lo = x - hi (exact, |lo| < 2^-10 |x|);
    the tensor core reads lo truncated to TF32 as well (error < 2^-10 |lo| < 2^-20 |x|).  Of the product a b = ah bh + ah bl + al bh + al bl
    the kernel computes ah bh + ah trunc(bl) + trunc(al) bh, exactly (TF32 x TF32 fits in fp32): the three neglected parts are each below
    2^-20 |a||b|.  They all have the sign of a b, so on all-positive data this error does not cancel;
  * K_chunk = 2 * 12 * min(K-blocks per split, kGemmChunk = 4) + (number of chunks per split), see `gemm_gamma`: the tensor core
    accumulates by truncation (up to 2^-23 = 2 * 2^-24 of the running sum per step) and one K-block is 4 K-steps x 3 MMAs = 12 steps,
    so a chunk has at most 48; each finished chunk is folded into the register accumulator with one round-to-nearest add;
  * splits: the fp32 sum of the split-K partials in `reduce_splits_kernel`; + 2: the final store and slack for the epilogue's fma.
  Every partial sum is bounded by (|A||B|^T)_ij, so this is a per-element bound whatever the data's signs and scales.
  Epilogue terms, each one rounding per operation:  out2 = fma(alpha, acc, bias): |alpha| times the bound of acc + 2^-24 (|alpha C| +
  |bias|);  affine  k0 acc + k1 E + k2 u_i u_j: |k0| times the bound of acc + 2^-24 (|k0 C| + 2 |k1 E| + 3 |k2 u_i u_j|).

Cholesky L L^T = A (`ops.cholesky`):  backward error |A - L L^T| <= C_ROUND_CHOL * 2^-24 * (n + 1) * |L||L|^T per element, and forward error
||L - L64||_F at most FWD_FACTOR times that of cuSOLVER (`torch.linalg.cholesky`, fp32) on the same fp32 input.

`emulate_gemm` is a float64 model of ideal 3xTF32 (bit truncation as the kernel does it) with the kernel's split-K plan (`plan_gemm`,
restated from the host code); the CPU tests show that it meets the bound and that every mutated variant -- single-pass TF32, lo x hi
dropped, the last K-block ignored, one split-K partial dropped, alpha (acc + bias), E transposed, u u^T dropped -- does not.  On the GPU
each case also checks the mutations on its own data, and asserts from the torch.profiler trace, taken in a child process
(`profiled_in_child`), the branch it claims: the
`gemm_tf32x3_kernel<CONVERT, false>` instance, the `split_tf32_kernel` / `lo_tf32_kernel` pre-passes, the split count (grid z) and
whether `reduce_splits_kernel` ran.  `emulate_cholesky` is the kernel's blocked algorithm (64 x 64 tiles, off-diagonal tiles through
the explicit inverse of the diagonal factor) in float64, with two mutations: one left-looking update skipped, inv(L_JJ) untransposed.

Non-finite inputs: a NaN or +-inf in A[i, k], B[j, k], E[i, j] or u_i makes exactly the elements non-finite that float64 does, and
every other element keeps the bits of the clean run.  The split turns +-inf into NaN (lo = inf - inf), so where float64 gives +-inf
the kernel gives NaN.
"""

import json
import math
import os
import re
import subprocess
import sys

import pytest
import torch

EPS = 2.0 ** -24
BM = BN = 128
BK = 32
CHUNK = 4  # kGemmChunk
SMS = 132  # kNumSMs: the split-K plan is fixed at build time, not read from the device
TF32_MASK = -8192  # 0xFFFFE000 as int32

# Calibrated once on an H100 80GB HBM3 (700 W); the data are seeded and the kernels deterministic, so these are fixed margins.
#   C_ROUND: the worst |err| / bound over every GEMM check here was 0.874 (X = sigma Y + m of the CMA-ES sampling product with a
#     diagonally scaled covariance), then 0.836 (383 x 383 x 31, scaled data, pre-split operands, affine epilogue) and 0.718 (the
#     active-weight SYRK at n = 4096, d = 1024); most cases stay below 0.36.  The mutations it must reject land at 6 and above.
#   C_ROUND_CHOL: the kernel's worst backward ratio was 0.456 (n = 33, cond 1e5; cuSOLVER 0.087 there, 0.122 at its worst): the
#     explicit 32 x 32 inverses cost up to ~5x cuSOLVER's componentwise residual at cond 1e5, inside the bound.
#   FWD_FACTOR: the kernel's forward error was at most 2.7 times cuSOLVER's (n = 1025, diagonally scaled by 1e+-3).
C_ROUND = 1.0
C_ROUND_CHOL = 1.0
FWD_FACTOR = 4.0


# ------------------------------------------------------------------------------------------------ plan and bound
def plan_gemm(M, N, K, allow_split=True):
    """(splits, K-blocks per split) of the host code's plan_gemm: split K while the grid stays within the SMs, at most 16 ways;
    the last split may be shorter, and rounding can leave fewer splits than the power of two chosen (5 K-blocks over 4 -> 3)."""
    tiles = -(-M // BM) * -(-N // BN)
    total_kb = -(-K // BK)
    splits = 1
    while allow_split and tiles * splits * 2 <= SMS and splits * 2 <= total_kb and splits < 16:
        splits *= 2
    kbps = -(-total_kb // splits)
    return -(-total_kb // kbps), kbps


def gemm_gamma(splits, kbps):
    k_chunk = 2 * 3 * (BK // 8) * min(kbps, CHUNK) + -(-kbps // CHUNK)
    return 3 * 2.0 ** -20 + EPS * (k_chunk + splits + 2)


def _split(x):
    """x (fp32) -> (hi, lo): hi = x with the 13 low mantissa bits cleared, lo = x - hi (exact)."""
    hi = (x.view(torch.int32) & TF32_MASK).view(torch.float32)
    return hi, x - hi


def _trunc(x):
    return (x.view(torch.int32) & TF32_MASK).view(torch.float32)


def emulate_gemm(A, B, splits, kbps, mutation=None):
    """A B^T as ideal 3xTF32 computes it: per split, hi*trunc(lo) + trunc(lo)*hi + hi*hi exactly, rounded to fp32, the partials summed
    in fp32.  `mutation`: hi_only, lo_hi_dropped, last_kblock_ignored, split_dropped."""
    ah, al = _split(A)
    bh, bl = _split(B)
    ah, al, bh, bl = ah.double(), _trunc(al).double(), bh.double(), _trunc(bl).double()
    K = A.shape[1]
    if mutation == "last_kblock_ignored":
        last = (-(-K // BK) - 1) * BK
        ah, al = ah.clone(), al.clone()
        ah[:, last:] = 0
        al[:, last:] = 0
    out = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float32, device=A.device)
    for s in range(splits):
        if mutation == "split_dropped" and s == splits - 1:  # (the first may cancel to zero on the `cancel` data)
            continue
        k0, k1 = s * kbps * BK, min(K, (s + 1) * kbps * BK)
        a_h, a_l, b_h, b_l = ah[:, k0:k1], al[:, k0:k1], bh[:, k0:k1], bl[:, k0:k1]
        part = a_h @ b_h.T
        if mutation != "hi_only":
            part = part + a_h @ b_l.T
            if mutation != "lo_hi_dropped":
                part = part + a_l @ b_h.T
        out = out + part.float()
    return out


def gemm_mutations(kind, splits):
    """The mutations of emulate_gemm the bound must reject on data of this kind.  On `scaled` data the K columns carry scales of
    2^-20..2^20, so a K range (the last K-block, one split) can weigh less than the bound and its loss is not an error one can see."""
    if kind == "scaled":
        return ["hi_only", "lo_hi_dropped"]
    return ["hi_only", "lo_hi_dropped", "last_kblock_ignored"] + (["split_dropped"] if splits > 1 else [])


def gemm_ref(A, B):
    """(A B^T, |A||B|^T) in float64."""
    A64, B64 = A.double(), B.double()
    return A64 @ B64.T, A64.abs() @ B64.abs().T


def epilogue(acc, absab, gamma, *, alpha=None, bias=None, k=None, E=None, u=None, mutation=None):
    """(value, bound) of the epilogue over acc (float64 A B^T, or a float64 / fp32 emulation), in float64.
    out2: alpha * acc + bias; affine: k0 acc + k1 E + k2 u u^T.  Mutations: alpha_bias (alpha (acc + bias)), E_transposed, uu_dropped."""
    acc = acc.double()
    bound = C_ROUND * gamma * absab
    if k is not None:
        k0, k1, k2 = (float(v) for v in k)
        E64 = torch.zeros_like(acc) if E is None else E.double()
        if mutation == "E_transposed":
            E64 = E64.T
        uu = torch.zeros_like(acc) if u is None or mutation == "uu_dropped" else torch.outer(u.double(), u.double())
        val = k0 * acc + k1 * E64 + k2 * uu
        bound = abs(k0) * bound + C_ROUND * EPS * (abs(k0) * acc.abs() + 2 * abs(k1) * E64.abs() + 3 * abs(k2) * uu.abs())
        return val, bound
    a = 1.0 if alpha is None else float(alpha)
    b = torch.zeros(acc.shape[1], dtype=torch.float64, device=acc.device) if bias is None else bias.double()
    val = a * (acc + b) if mutation == "alpha_bias" else a * acc + b
    bound = abs(a) * bound + C_ROUND * EPS * (abs(a) * acc.abs() + b.abs())
    return val, bound


def ratio(y, ref, bound):
    """Worst |y - ref| / bound (inf if y is non-finite where ref is finite)."""
    err = (y.double() - ref).abs()
    r = err / bound.clamp_min(1e-300)
    r = torch.where(torch.isfinite(err), r, torch.full_like(r, math.inf))
    return float(r.max())


def within(y, ref, bound):
    return bool(((y.double() - ref).abs() <= bound).all())  # NaN compares False


# ------------------------------------------------------------------------------------------------ data
def make_data(kind, rows, K, seed):
    """fp32 (rows, K) on the CPU: randn; positive (uniform [0, 1): the truncation errors all have one sign); scaled (rows and columns
    scaled by powers of two over 2^-20..2^20 each, elements over 2^-40..2^40); cancel (the second half of K repeats the first with a relative
    2^-6 perturbation, in the B operand with its sign flipped: C ~ 2^-6 of |A||B|^T, and the truncation errors of the two halves do
    not cancel each other as they would on an exact mirror)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "positive":
        return torch.rand(rows, K, generator=g)
    x = torch.randn(rows, K, generator=g)
    if kind == "scaled":
        re_ = torch.randint(-20, 21, (rows, 1), generator=g).float()
        ce = torch.randint(-20, 21, (1, K), generator=g).float()
        x = x * torch.exp2(re_) * torch.exp2(ce)
    return x


def make_pair(kind, M, N, K, seed):
    if kind != "cancel":
        return make_data(kind, M, K, seed), make_data(kind, N, K, seed + 1)
    h = K // 2
    A, B = make_data("randn", M, K, seed), make_data("randn", N, K, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    A[:, h:2 * h] = A[:, :h] * (1 + 2.0 ** -6 * torch.randn(M, h, generator=g))
    B[:, h:2 * h] = -B[:, :h] * (1 + 2.0 ** -6 * torch.randn(N, h, generator=g))
    return A, B


def spd(n, cond, seed, scale=None):
    """fp32 symmetric positive definite Q diag(lambda) Q^T (lambda log-spaced over 1..cond), optionally scaled S R S by a diagonal
    S = logspace(-scale, scale); symmetrised exactly in fp32."""
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(n, n, generator=g, dtype=torch.float64))
    lam = torch.logspace(0, math.log10(cond), n, dtype=torch.float64)
    a = (q * lam) @ q.T
    if scale is not None:
        s = torch.logspace(-scale, scale, n, dtype=torch.float64)[torch.randperm(n, generator=g)]
        a = s[:, None] * a * s[None, :]
    a = a.float()
    return torch.tril(a) + torch.tril(a, -1).T


def cmaes_factor(d, seed, kind):
    """The sampling factor A of CMA-ES: chol(Q diag(lambda) Q^T), lambda log-spaced over 1..1e6, or chol(S R S) with a well-conditioned
    correlation R and S over 1e-3..1e3."""
    if kind == "ill":
        c = spd(d, 1e6, seed).double()
    else:
        g = torch.Generator().manual_seed(seed)
        b = torch.randn(d, d, generator=g, dtype=torch.float64)
        r = b @ b.T / d + torch.eye(d, dtype=torch.float64)
        r = r / torch.sqrt(torch.outer(r.diagonal(), r.diagonal()))
        s = torch.logspace(-3, 3, d, dtype=torch.float64)[torch.randperm(d, generator=g)]
        c = s[:, None] * r * s[None, :]
    return torch.linalg.cholesky(c).float().contiguous()


def cmaes_weights(n, d):
    """The active CMA-ES weights of cmaes.py for popsize n, dimension d (positive part sums to 1, negative part scaled by alpha), and
    (c_1, c_mu)."""
    mu = n // 2
    raw = math.log((n + 1) / 2) - torch.log(torch.arange(n, dtype=torch.float64) + 1)
    pos, neg = raw[:mu], raw[mu:]
    mu_eff = float(pos.sum() ** 2 / (pos ** 2).sum())
    c_1 = min(1, n / 6) * 2 / ((d + 1.3) ** 2.0 + mu_eff)
    c_mu = min(1 - c_1, 2 * ((0.25 + mu_eff - 2 + (1 / mu_eff)) / ((d + 2) ** 2.0 + mu_eff)))
    mu_eff_neg = float(neg.sum() ** 2 / (neg ** 2).sum())
    alpha = min(1 + c_1 / c_mu, 1 + 2 * mu_eff_neg / (mu_eff + 2), (1 - c_mu - c_1) / (d * c_mu))
    return torch.cat([pos / pos.sum(), alpha * neg / neg.abs().sum()]), c_1, c_mu


# ------------------------------------------------------------------------------------------------ Cholesky emulation
def emulate_cholesky(A, mutation=None, nb=64):
    """The kernel's blocked left-looking algorithm in float64: tile (I, J) = A[I, J] - sum_{k<J} L[I, k] L[J, k]^T; a diagonal tile is
    factorised, an off-diagonal one multiplied by inv(L[J, J])^T.  Mutations: update_skipped (the k = 0 update of tile (2, 1)),
    inv_untransposed."""
    A = A.double()
    n = A.shape[0]
    T = -(-n // nb)
    L = torch.zeros_like(A)
    sl = [slice(t * nb, min(n, (t + 1) * nb)) for t in range(T)]
    for J in range(T):
        for I in range(J, T):
            t = torch.tril(A[sl[I], sl[J]]) + torch.tril(A[sl[I], sl[J]], -1).T if I == J else A[sl[I], sl[J]].clone()
            for k in range(J):
                if mutation == "update_skipped" and (I, J, k) == (2, 1, 0):
                    continue
                t = t - L[sl[I], sl[k]] @ L[sl[J], sl[k]].T
            if I == J:
                f, info = torch.linalg.cholesky_ex(t)  # (a mutation can leave a tile that is not positive definite: NaN, like the kernel)
                L[sl[J], sl[J]] = f if int(info) == 0 else math.nan
            else:
                inv = torch.linalg.inv(L[sl[J], sl[J]])
                L[sl[I], sl[J]] = t @ (inv if mutation == "inv_untransposed" else inv.T)
    return L


def chol_backward(A, L):
    """(|A - L L^T|, |L||L|^T) in float64."""
    L64 = L.double()
    return (A.double() - L64 @ L64.T).abs(), L64.abs() @ L64.abs().T


def chol_ratio(A, L):
    """Worst |A - L L^T| / (2^-24 (n + 1) |L||L|^T) (C_ROUND_CHOL = 1)."""
    res, mag = chol_backward(A, L)
    if not bool(torch.isfinite(L).all()):
        return math.inf
    return float((res / (EPS * (A.shape[0] + 1) * mag).clamp_min(1e-300)).max())


# ================================================================================================ CPU: the bound and its oracle
CPU_CASES = [  # (M, N, K, data)
    (4, 127, 3, "randn"), (33, 40, 129, "positive"), (128, 128, 33, "cancel"), (20, 24, 1000, "scaled"), (16, 16, 4099, "positive"),
]


@pytest.mark.parametrize("M,N,K,kind", CPU_CASES)
def test_emulation_meets_the_bound_and_mutations_do_not(M, N, K, kind):
    A, B = make_pair(kind, M, N, K, seed=M + N + K)
    splits, kbps = plan_gemm(M, N, K)
    gamma = gemm_gamma(splits, kbps)
    ref, absab = gemm_ref(A, B)
    y = emulate_gemm(A, B, splits, kbps)
    assert within(y, ref, C_ROUND * gamma * absab), ratio(y, ref, C_ROUND * gamma * absab)
    for m in gemm_mutations(kind, splits):
        assert not within(emulate_gemm(A, B, splits, kbps, m), ref, C_ROUND * gamma * absab), m


def test_epilogue_mutations_are_rejected():
    A, B = make_pair("randn", 64, 64, 96, seed=5)
    splits, kbps = plan_gemm(64, 64, 96)
    gamma = gemm_gamma(splits, kbps)
    ref, absab = gemm_ref(A, B)
    y = emulate_gemm(A, B, splits, kbps)
    g = torch.Generator().manual_seed(6)
    bias, E, u = torch.randn(64, generator=g), torch.randn(64, 64, generator=g), torch.randn(64, generator=g)
    kw = dict(alpha=torch.tensor(0.3), bias=bias)
    v, b = epilogue(y, absab, gamma, **kw)
    r, _ = epilogue(ref, absab, gamma, **kw)
    assert within(v.float(), r, b)
    assert not within(epilogue(y, absab, gamma, mutation="alpha_bias", **kw)[0].float(), r, b)
    kw = dict(k=(0.75, 1.25, -0.5), E=E, u=u)
    v, b = epilogue(y, absab, gamma, **kw)
    r, _ = epilogue(ref, absab, gamma, **kw)
    assert within(v.float(), r, b)
    for m in ("E_transposed", "uu_dropped"):
        assert not within(epilogue(y, absab, gamma, mutation=m, **kw)[0].float(), r, b), m


@pytest.mark.parametrize("M,N,K,splits,kbps", [
    (128, 128, 33, 2, 1), (128, 128, 129, 3, 2), (128, 128, 128, 4, 1), (383, 383, 1000, 8, 4), (128, 128, 1000, 16, 2),
    (383, 383, 4099, 8, 17), (129, 129, 4099, 15, 9), (1, 4, 1, 1, 1), (1025, 1025, 4096, 1, 128), (1024, 1024, 4096, 2, 64),
])
def test_plan_gemm_split_counts(M, N, K, splits, kbps):
    assert plan_gemm(M, N, K) == (splits, kbps)


def test_cholesky_emulation_meets_the_bound_and_mutations_do_not():
    A = spd(200, 1e4, seed=3)
    assert chol_ratio(A, emulate_cholesky(A).float()) <= C_ROUND_CHOL
    for m in ("update_skipped", "inv_untransposed"):
        assert chol_ratio(A, emulate_cholesky(A, m).float()) > C_ROUND_CHOL, m


# ================================================================================================ GPU: GEMM
KNAME = re.compile(r"gemm_tf32x3_kernel<(true|false), (true|false)>")


def profile_kernels(run):
    """[(kernel name, grid)] of the kernels `run` launches, in launch order."""
    import tempfile

    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        for _ in range(3):  # now and then the profiler delivers no kernel record from a short window: take another
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            prof.export_chrome_trace(path)
            with open(path) as f:
                evs = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
            if evs:
                break
    assert evs, "no kernel record"
    return [(e["name"], tuple(e["args"]["grid"])) for e in sorted(evs, key=lambda e: e["ts"])]


def branch_of(launches):
    """(CONVERT, split count = grid z of the GEMM, split_tf32_kernel launches, lo_tf32_kernel launches, reduce_splits_kernel launches)."""
    gem = [(KNAME.search(n), g) for n, g in launches if "gemm_tf32x3_kernel" in n]
    assert len(gem) == 1 and gem[0][0] and gem[0][0].group(2) == "false", launches
    count = lambda s: sum(s in n for n, _ in launches)  # noqa: E731
    return (gem[0][0].group(1) == "true", gem[0][1][2], count("split_tf32_kernel"), count("lo_tf32_kernel"),
            count("reduce_splits_kernel"))


def place(x, layout, dev="cuda"):
    """x (rows, K) on the device with a layout: aligned (16-byte base, pitch K rounded up to 4: TMA-addressable), offset (one float
    past a 16-byte boundary), pitch (pitch a multiple of 4 plus 1), contig (pitch K).  Unused elements are NaN."""
    rows, K = x.shape
    ld = {"aligned": -(-K // 4) * 4, "offset": -(-K // 4) * 4, "pitch": -(-K // 4) * 4 + 1, "contig": K}[layout]
    off = 1 if layout == "offset" else 0
    buf = torch.full((rows * ld + 8,), math.nan, dtype=torch.float32, device=dev)
    v = buf[off:off + rows * ld].view(rows, ld)[:, :K]
    v.copy_(x)
    return v


def tma_ok(t):
    return t.data_ptr() % 16 == 0 and t.stride(0) % 4 == 0


def gemm_affine(A, B, k, E=None, u=None, out=None):
    """evok_gemm_nt_affine: out = k0 A B^T + k1 E + k2 u u^T on any operand layout (ops.weighted_syrk_update only makes aligned ones)."""
    from evotorch_b200 import _native as nat

    M, N, K = A.shape[0], B.shape[0], A.shape[1]
    out = torch.empty(M, N, device=A.device) if out is None else out
    lib = nat.lib()
    ws = nat.workspace(A.device, lib.evok_gemm_workspace_bytes(M, N, K), "gemm")
    nat.check(lib.evok_gemm_nt_affine(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), M, N, K, out.data_ptr(), out.stride(0),
                                      k.data_ptr(), nat.ptr(E), 0 if E is None else E.stride(0), nat.ptr(u), ws.data_ptr(), ws.numel(),
                                      nat.stream_of(A)), "evok_gemm_nt_affine")
    return out


# (id, M, N, K, A layout, B layout, C layout, data, epilogue).  The comment gives the plan: splits x K-blocks per split.
GEMM_CASES = [
    ("1x4x1", 1, 4, 1, "aligned", "aligned", "aligned", "randn", None),  # 1 x 1
    ("4x127x3_presplit", 4, 127, 3, "contig", "contig", "offset", "positive", None),  # 1 x 1, pitch 3
    ("127x129x31", 127, 129, 31, "aligned", "aligned", "offset", "scaled", None),  # 1 x 1, N % 4 != 0, C unaligned
    ("128x128x33_presplit", 128, 128, 33, "contig", "contig", "aligned", "cancel", None),  # 2 x 1
    ("128x128x129_short", 128, 128, 129, "aligned", "aligned", "aligned", "positive", None),  # 3 x 2, last split 1 K-block
    ("128x128x128_aoff", 128, 128, 128, "offset", "aligned", "aligned", "randn", None),  # 4 x 1, pre-split (A one float in)
    ("383x129x160", 383, 129, 160, "aligned", "pitch", "offset", "scaled", None),  # 3 x 2, pre-split (B pitch 161)
    ("383x383x1000", 383, 383, 1000, "aligned", "aligned", "aligned", "positive", None),  # 8 x 4
    ("128x128x1000", 128, 128, 1000, "aligned", "aligned", "offset", "cancel", None),  # 16 x 2
    ("383x383x4099", 383, 383, 4099, "aligned", "aligned", "aligned", "positive", None),  # 8 x 17: chunk boundaries in a split
    ("129x129x4099_presplit", 129, 129, 4099, "contig", "contig", "aligned", "scaled", None),  # 15 x 9, last split 3 K-blocks
    ("129x383x4099_out2", 129, 383, 4099, "aligned", "aligned", "aligned", "positive", "out2_ab"),  # 1 x 129: 33 chunks in one CTA
    ("383x4x127_out2", 383, 4, 127, "offset", "contig", "offset", "randn", "out2_ab"),  # 1 x 4
    ("1x129x1000_out2", 1, 129, 1000, "aligned", "aligned", "aligned", "scaled", "out2_a"),
    ("128x127x32_out2", 128, 127, 32, "aligned", "aligned", "offset", "cancel", "out2_b"),
    ("127x1x33_out2", 127, 1, 33, "aligned", "pitch", "aligned", "randn", "out2"),
    ("129x129x32_k", 129, 129, 32, "aligned", "aligned", "aligned", "randn", "k"),  # affine in the epilogue
    ("129x129x1000_k", 129, 129, 1000, "aligned", "aligned", "aligned", "positive", "k"),  # 16 x 2: affine in the reduction
    ("383x383x31_kE", 383, 383, 31, "offset", "aligned", "offset", "scaled", "kE"),
    ("383x383x1000_kE", 383, 383, 1000, "aligned", "pitch", "aligned", "randn", "kE"),
    ("127x127x32_kEu", 127, 127, 32, "aligned", "aligned", "aligned", "cancel", "kEu"),
    ("128x128x129_kEu", 128, 128, 129, "contig", "aligned", "offset", "randn", "kEu"),
    ("383x383x32_inplace", 383, 383, 32, "aligned", "aligned", "aligned", "positive", "kEu_inplace"),
    ("128x128x4099_inplace", 128, 128, 4099, "aligned", "aligned", "aligned", "randn", "kE_inplace"),  # 15 x 9
]
B_LO_TMA_CASES = ["127x129x31", "128x128x129_short", "383x383x4099", "129x383x4099_out2", "128x128x1000"]


def run_gemm_case(case_id, check_mutations=True, profiled=False):
    """Runs one GEMM_CASES entry; returns {ratio, splits, kbps} and, `profiled`, {convert, grid_z, presplit, lo_tma, reduce, kernels}
    from the torch.profiler trace.  Asserts the bound, the mutations (on this case's data) and, `profiled`, that the branch it ran is
    the one the plan says."""
    _, M, N, K, la, lb, lc, kind, epi = next(c for c in GEMM_CASES if c[0] == case_id)
    from evotorch_b200 import ops

    A_cpu, B_cpu = make_pair(kind, M, N, K, seed=M * 7 + N * 3 + K)
    A, B = place(A_cpu, la), place(B_cpu, lb)
    g = torch.Generator().manual_seed(K)
    out = place(torch.zeros(M, N), lc)
    kw = {}
    affine = epi is not None and epi.startswith("k")
    if epi and epi.startswith("out2"):
        out2 = place(torch.zeros(M, N), "offset" if lc == "aligned" else "aligned")
        kw = dict(alpha=torch.tensor([0.3]).cuda() if "a" in epi[4:] else None, bias=torch.randn(N, generator=g).cuda() if "b" in epi[4:] else None)
        run = lambda: ops.gemm_nt(A, B, out, out2=out2, **kw)  # noqa: E731
    elif affine:
        E = u = None
        if "E" in epi:
            E = torch.randn(M, N, generator=g).cuda() * (1 - 2 * torch.rand(M, N, generator=g).cuda())  # not symmetric
            if "inplace" in epi:
                out.copy_(E)
                E = out
        if "u" in epi:
            u = torch.randn(M, generator=g).cuda()
        k = torch.tensor([0.75, 1.25, -0.5]).cuda()
        E0 = None if E is None else E.clone()
        kw = dict(k=k.cpu(), E=E0, u=u)
        run = lambda: gemm_affine(A, B, k, E=E, u=u, out=out)  # noqa: E731
    else:
        run = lambda: ops.gemm_nt(A, B, out)  # noqa: E731
    splits, kbps = plan_gemm(M, N, K, allow_split=not (epi or "").startswith("out2"))
    res = dict(splits=splits, kbps=kbps)
    if profiled:
        names = profile_kernels(run)
        convert, grid_z, n_split, n_lo, n_reduce = branch_of(names)
        b_lo_tma = os.environ.get("EVOK_GEMM_B_LO_TMA", "0") == "1"
        assert convert == (tma_ok(A) and tma_ok(B)), (case_id, names)
        assert grid_z == splits, (case_id, names)
        assert n_split == (0 if convert else 2), (case_id, names)
        assert n_lo == (1 if convert and b_lo_tma else 0), (case_id, names)
        assert n_reduce == (1 if splits > 1 else 0), (case_id, names)
        res.update(convert=convert, grid_z=grid_z, presplit=n_split, lo_tma=n_lo, reduce=n_reduce,
                   kernels=[n.split("(")[0] for n, _ in names])
    else:
        run()
    gamma = gemm_gamma(splits, kbps)
    ref, absab = gemm_ref(A_cpu.cuda(), B_cpu.cuda())
    y = out
    if epi and epi.startswith("out2"):
        acc_v, acc_b = epilogue(ref, absab, gamma)
        assert within(out, acc_v, acc_b), ratio(out, acc_v, acc_b)
        ref, bound = epilogue(ref, absab, gamma, **kw)
        y = out2
    elif affine:
        ref, bound = epilogue(ref, absab, gamma, **kw)
    else:
        bound = C_ROUND * gamma * absab
    r = ratio(y, ref, bound)
    print(f"{case_id}: |err| / bound {r:.3g}, {splits} x {kbps} K-blocks")
    assert r <= 1.0, f"{case_id}: worst |err| / bound {r:.3g}"
    if check_mutations:
        emu = emulate_gemm(A_cpu.cuda(), B_cpu.cuda(), splits, kbps)
        for m in gemm_mutations(kind, splits):
            y_m = emulate_gemm(A_cpu.cuda(), B_cpu.cuda(), splits, kbps, m)
            if epi:
                y_m = epilogue(y_m, absab, gamma, **kw)[0].float()
            assert not within(y_m, ref, bound), f"{case_id}: the bound does not reject {m}"
        epi_muts = {"out2_ab": ["alpha_bias"], "kE": ["E_transposed"], "kEu": ["E_transposed", "uu_dropped"],
                    "kEu_inplace": ["E_transposed", "uu_dropped"], "kE_inplace": ["E_transposed"]}.get(epi, [])
        for m in epi_muts:
            assert not within(epilogue(emu, absab, gamma, mutation=m, **kw)[0].float(), ref, bound), f"{case_id}: {m} not rejected"
    res["ratio"] = r
    return res


_CHILD = """
import json, sys, traceback
sys.path[:0] = [%r, %r]
import test_matrix_kernels as t
out = {}
for c in %r:
    try:
        out[c] = t.run_gemm_case(c, check_mutations=False, profiled=True)
    except Exception:
        out[c] = {"error": traceback.format_exc()[-2000:]}
print("RESULT", json.dumps(out))
"""


def profiled_in_child(cases, b_lo_tma):
    """{case id: run_gemm_case(..., profiled=True) or {error}} from a child process.  The profiler runs there, never in the test
    process: a CUPTI session that ends in a process is torn down, and the re-initialised one of a later profiler window in the same
    process (another test file's) can come back without kernel records.  EVOK_GEMM_B_LO_TMA is read once per process as well."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, EVOK_GEMM_B_LO_TMA="1" if b_lo_tma else "0")
    p = subprocess.run([sys.executable, "-c", _CHILD % (os.path.dirname(here), here, list(cases))], env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    return json.loads(next(line for line in p.stdout.splitlines() if line.startswith("RESULT "))[7:])


@pytest.fixture(scope="module")
def branches():
    return profiled_in_child([c[0] for c in GEMM_CASES], b_lo_tma=False)


@pytest.mark.gpu
@pytest.mark.parametrize("case_id", [c[0] for c in GEMM_CASES])
def test_gemm_case(case_id, branches):
    """The bound and the mutations here; the branch (and the bound once more) under the profiler in a child process."""
    run_gemm_case(case_id)
    res = branches[case_id]
    assert "error" not in res, res.get("error")
    print(f"{case_id}: kernels {res['kernels']}, grid z {res['grid_z']}")


@pytest.mark.gpu
def test_gemm_b_lo_tma_in_a_subprocess():
    """EVOK_GEMM_B_LO_TMA=1: B's lo tile from a pre-split copy by TMA (`lo_tf32_kernel` + the CONVERT kernel)."""
    res = profiled_in_child(B_LO_TMA_CASES, b_lo_tma=True)
    print("EVOK_GEMM_B_LO_TMA=1:", res)
    assert all("error" not in r for r in res.values()), res
    assert all(r["convert"] and r["lo_tma"] == 1 for r in res.values()), res


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(129, 129, 32), (128, 128, 1000)])
def test_gemm_non_finite_inputs(M, N, K):
    """NaN / +-inf in A, B, E and u: exactly float64's non-finite elements, every other element bit-identical to the clean run."""
    A, B = make_pair("randn", M, N, K, seed=11)
    g = torch.Generator().manual_seed(12)
    E, u = torch.randn(M, N, generator=g), torch.randn(M, generator=g)
    k = torch.tensor([0.75, 1.25, -0.5]).cuda()
    clean = gemm_affine(A.cuda(), B.cuda(), k, E=E.cuda(), u=u.cuda()).clone()
    An, Bn, En, un = A.clone(), B.clone(), E.clone(), u.clone()
    An[3, 5], An[70, K - 1], Bn[9, 0], Bn[100, K // 2] = math.nan, math.inf, -math.inf, math.nan
    En[20, 40], un[60] = math.inf, math.nan
    y = gemm_affine(An.cuda(), Bn.cuda(), k, E=En.cuda(), u=un.cuda()).cpu()
    prod = (An.double()[:, None, :] * Bn.double()[None, :, :]).sum(-1)  # element-wise IEEE arithmetic: no BLAS zero skipping
    ref = 0.75 * prod + 1.25 * En.double() + -0.5 * torch.outer(un.double(), un.double())
    bad = torch.zeros(M, N, dtype=torch.bool)
    bad[[3, 70], :] = True
    bad[:, [9, 100]] = True
    bad[20, 40] = True
    bad[60, :] = True
    bad[:, 60] = True
    assert torch.equal(~torch.isfinite(ref), bad)
    assert torch.equal(~torch.isfinite(y), bad)
    assert torch.equal(y[~bad].view(torch.int32), clean.cpu()[~bad].view(torch.int32))
    # the split turns +-inf into NaN: rows / columns reached only through an infinite operand come out NaN, not +-inf
    assert bool(torch.isnan(y[70, :]).all()) and bool(torch.isnan(y[:, 9]).all())


# Both operands times s = 2^e: the results scale exactly (the same worst ratio, 0.046, at every e) down to e = -60, where the products
# are ~2^-120 and the lo x hi corrections ~2^-131 -- the correction terms do not underflow on their own.  At e = -64 the ratio is 0.056;
# at e = -68 (8.0) and below the results themselves are fp32 subnormals, which carry no relative accuracy.  So the bound is asserted
# down to SCALE_FLOOR and the sweep goes on to -76 only to show where it stops holding.
SCALE_FLOOR = -64


@pytest.mark.gpu
def test_gemm_scale_sweep():
    from evotorch_b200 import ops

    A, B = make_pair("randn", 128, 128, 256, seed=21)
    ratios = {}
    for e in range(0, -77, -4):
        s = 2.0 ** e
        As, Bs = (A * s).cuda(), (B * s).cuda()
        y = ops.gemm_nt(As, Bs)
        splits, kbps = plan_gemm(128, 128, 256)
        ref, absab = gemm_ref(As, Bs)
        ratios[e] = ratio(y, ref, C_ROUND * gemm_gamma(splits, kbps) * absab)
    print("scale sweep |err| / bound:", ratios)
    assert all(r <= 1.0 for e, r in ratios.items() if e >= SCALE_FLOOR), ratios


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ill", "scaled"])
def test_gemm_cmaes_sampling_operands(kind):
    """Y = Z A^T with the sampling factor of an ill-conditioned or badly scaled covariance, and X = sigma Y + m in out2."""
    from evotorch_b200 import ops

    d, n = 383, 129
    Af = cmaes_factor(d, seed=31, kind=kind)
    g = torch.Generator().manual_seed(32)
    Z = torch.randn(n, d, generator=g)
    m = torch.randn(d, generator=g)
    sigma = torch.tensor([0.37])
    Y, X = torch.empty(n, d, device="cuda"), torch.empty(n, d, device="cuda")
    ops.gemm_nt(Z.cuda(), Af.cuda(), Y, out2=X, alpha=sigma.cuda(), bias=m.cuda())
    splits, kbps = plan_gemm(n, d, d, allow_split=False)
    gamma = gemm_gamma(splits, kbps)
    ref, absab = gemm_ref(Z.cuda(), Af.cuda())
    xr, xb = epilogue(ref, absab, gamma, alpha=sigma, bias=m.cuda())
    r = (ratio(Y, ref, C_ROUND * gamma * absab), ratio(X, xr, xb))
    print(f"CMA-ES sampling ({kind}): |err| / bound Y {r[0]:.3g}, X {r[1]:.3g}")
    assert max(r) <= 1.0, r


def _syrk_check(Y, w, k, C, u, pre_round=True):
    from evotorch_b200 import ops

    n, d = Y.shape
    out = ops.weighted_syrk_update(Y.cuda(), w.float().cuda(), k.cuda(), C.cuda(), None if u is None else u.cuda())
    splits, kbps = plan_gemm(d, d, n)
    gamma = gemm_gamma(splits, kbps) + EPS  # + the rounding of w_r Y_rc in the transposing pass
    w32 = w.float().cuda().double()
    Y64 = Y.cuda().double()
    acc = (Y64 * w32[:, None]).T @ Y64
    absab = (Y64.abs() * w32.abs()[:, None]).T @ Y64.abs()
    ref, bound = epilogue(acc, absab, gamma, k=k, E=C.cuda(), u=None if u is None else u.cuda())
    return ratio(out, ref, bound), splits


@pytest.mark.gpu
def test_syrk_cmaes_active_weights():
    """The rank-mu + rank-1 covariance update of CMA-ES at n = 4096, d = 1024, with active weights and an ill-conditioned C."""
    n, d = 4096, 1024
    w, c_1, c_mu = cmaes_weights(n, d)
    Af = cmaes_factor(d, seed=41, kind="ill")
    g = torch.Generator().manual_seed(42)
    Z = torch.randn(n, d, generator=g)
    Y = (Z.cuda() @ Af.cuda().T).cpu()  # any fp32 Y will do: the check is against float64 of this Y
    neg = w < 0
    w = torch.where(neg, d * w / (Z.double() ** 2).sum(1), w)
    C = (Af.double() @ Af.double().T).float()
    u = torch.randn(d, generator=g) * 0.1
    k = torch.tensor([c_mu, 1 - c_1 - c_mu * float(w.sum()), c_1], dtype=torch.float32)
    r, splits = _syrk_check(Y, w, k, C, u)
    print(f"CMA-ES SYRK n={n} d={d}: |err| / bound {r:.3g}")
    assert splits == 2
    assert r <= 1.0, r


@pytest.mark.gpu
def test_syrk_xnes_centred_weights():
    """XNES: Z^T diag(w) Z - sum(w) I with zero-sum (centred) utility weights: the sum cancels."""
    n, d = 1000, 129
    g = torch.Generator().manual_seed(51)
    Z = torch.randn(n, d, generator=g)
    util = torch.clamp(math.log(n / 2 + 1) - torch.log(torch.arange(1, n + 1, dtype=torch.float64)), min=0)
    w = util / util.sum() - 1.0 / n
    k = torch.tensor([1.0, -float(w.float().sum()), 0.0])
    r, splits = _syrk_check(Z, w, k, torch.eye(d), None)
    print(f"XNES SYRK n={n} d={d}: |err| / bound {r:.3g}")
    assert splits == 16
    assert r <= 1.0, r


# ================================================================================================ GPU: Cholesky
CHOL_N = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 1024, 1025]
CHOL_CASES = [(n, c) for n in CHOL_N for c in (1e2, 1e4)] + [(n, 1e5) for n in CHOL_N if n <= 256]


def _chol_check(A, mutations=True):
    from evotorch_b200 import ops

    n = A.shape[0]
    L = ops.cholesky(A.cuda()).cpu()
    Lcu, info = torch.linalg.cholesky_ex(A.cuda())
    L64 = torch.linalg.cholesky(A.double())
    r = chol_ratio(A, L)
    r_cu = chol_ratio(A, Lcu.cpu()) if int(info) == 0 else math.inf
    fwd = float(torch.linalg.norm(L.double() - L64))
    fwd_cu = float(torch.linalg.norm(Lcu.cpu().double() - L64)) if int(info) == 0 else math.inf
    if mutations and n > 128:
        for m in ("update_skipped", "inv_untransposed"):
            assert chol_ratio(A, emulate_cholesky(A, m).float()) > C_ROUND_CHOL, m
    return r, r_cu, fwd, fwd_cu


@pytest.mark.gpu
@pytest.mark.parametrize("n,cond", CHOL_CASES)
def test_cholesky_conditioned(n, cond):
    A = spd(n, cond, seed=n)
    r, r_cu, fwd, fwd_cu = _chol_check(A, mutations=cond == 1e4)
    if r_cu == math.inf:
        pytest.skip("cuSOLVER fp32 fails on this input")
    print(f"n={n} cond={cond:g}: backward {r:.3g} (cuSOLVER {r_cu:.3g}), forward {fwd:.3g} (cuSOLVER {fwd_cu:.3g})")
    assert r <= C_ROUND_CHOL, (r, r_cu)
    assert fwd <= FWD_FACTOR * fwd_cu + 1e-300, (fwd, fwd_cu)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [65, 200, 1025])
def test_cholesky_diagonally_scaled(n):
    A = spd(n, 10.0, seed=n + 1, scale=3)
    r, r_cu, fwd, fwd_cu = _chol_check(A)
    print(f"n={n} scaled: backward {r:.3g} (cuSOLVER {r_cu:.3g}), forward {fwd:.3g} (cuSOLVER {fwd_cu:.3g})")
    assert r <= C_ROUND_CHOL, (r, r_cu)
    assert fwd <= FWD_FACTOR * fwd_cu, (fwd, fwd_cu)


@pytest.mark.gpu
def test_cholesky_of_a_syrk_covariance():
    """The covariance CMA-ES factorises: C' = weighted_syrk_update(...) of an ill-conditioned C, from the kernels themselves."""
    from evotorch_b200 import ops

    n, d = 4096, 200
    w, c_1, c_mu = cmaes_weights(n, d)
    w = w.clamp_min(0)  # positive weights: C' stays positive definite
    Af = cmaes_factor(d, seed=61, kind="ill")
    g = torch.Generator().manual_seed(62)
    Y = torch.randn(n, d, generator=g).cuda() @ Af.cuda().T
    C = (Af.double() @ Af.double().T).float().cuda()
    k = torch.tensor([c_mu, 1 - c_1 - c_mu * float(w.sum()), c_1]).cuda()
    Cn = ops.weighted_syrk_update(Y, w.float().cuda(), k, C, torch.randn(d, generator=g).cuda() * 0.1).cpu()
    Cn = torch.tril(Cn) + torch.tril(Cn, -1).T
    r, r_cu, fwd, fwd_cu = _chol_check(Cn)
    print(f"syrk covariance: backward {r:.3g} (cuSOLVER {r_cu:.3g}), forward {fwd:.3g} (cuSOLVER {fwd_cu:.3g})")
    assert r <= C_ROUND_CHOL, (r, r_cu)
    assert fwd <= FWD_FACTOR * fwd_cu, (fwd, fwd_cu)


@pytest.mark.gpu
def test_cmaes_with_the_kernel_cholesky(monkeypatch):
    """CMAES with EVOTORCH_B200_EVOK_CHOLESKY=1 on a 1e6 ellipsoid: every factor it computes meets the backward bound against the
    covariance it was computed from."""
    from evotorch_b200 import Problem
    from evotorch_b200.algorithms import CMAES

    monkeypatch.setenv("EVOTORCH_B200_EVOK_CHOLESKY", "1")
    d = 66  # two 64-wide block columns: off-diagonal tiles and left-looking updates
    scale = torch.logspace(0, 6, d, device="cuda")
    prob = Problem("min", lambda x: (x * x * scale).sum(-1), initial_bounds=(-3, 3), solution_length=d, device="cuda", seed=3,
                   vectorized=True)
    c = CMAES(prob, stdev_init=1.0)
    worst, checked = 0.0, 0
    for _ in range(1500):
        A0 = c.A.clone()
        c.step()
        if not torch.equal(A0, c.A):
            C = c.C.cpu()
            C = torch.tril(C) + torch.tril(C, -1).T  # the kernel reads the lower triangle
            worst = max(worst, chol_ratio(C, c.A.cpu()))
            checked += 1
    cond = float(torch.linalg.cond(c.C.double()))
    print(f"CMAES + kernel Cholesky: {checked} factorisations, final cond(C) {cond:.3g}, worst backward ratio {worst:.3g}")
    assert checked > 10
    assert worst <= C_ROUND_CHOL, worst
