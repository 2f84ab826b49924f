"""The shared-minibatch policy forward, branch by branch, against a float64 evaluation of the same fp32 parameters.

`ops.mlp_forward_shared` (behind `Policy.forward_shared` and `NEProblem.batched_forward`) runs in two steps (csrc/evok_mlp.cu):
  * layer 1 of all N networks is one gather GEMM (`gemm_gather_persistent_kernel`, 3xTF32 on wgmma) whose epilogue applies bias and
    activation, one instantiation per activation;
  * layers 2..n run in `mlp_tail2_kernel<OG>` when n_layers == 2, dout <= 32, h1 % 4 == 0 and its shared memory,
    (96 h1 + 2336) floats, fits in 200 KB -- h1 <= 508 (204 416 B), while h1 = 512 needs 205 952 B -- with OG = 1, 2, 4, 5, 8 from
    ceil(dout / 4); in `mlp_tail_kernel` otherwise;
  * the population goes through in chunks of 2^30 / (h1 * ldh * 4) networks, ldh = B rounded up to a multiple of 4.
The gather GEMM is also called directly through the C ABI (`evok_gemm_gather_rows`, `evok_gemm_gather_rows_ws`), and the per-policy
forward `ops.mlp_forward` (K8) is checked at its limits against the same oracle.

Tolerance, per element:  |y - y64| <= C_ROUND * 2^-24 * K_eff * mag + aerr  with
  * mag:  the same net evaluated in float64 on |W|, |b|, |x| with identity activations.  Every activation used is 1-Lipschitz, so an
          error e in the input of a layer moves its output by at most |W| e: mag bounds what rounding can reach in every output;
  * K_eff: the largest fan-in of the net;
  * aerr: ACT_ERR for every tanh / sigmoid unit (tanh_abs1e7 in the GEMM epilogue, tanh_1e6 and the __expf sigmoid in the tail
          kernels, all within about 1e-6 absolute), propagated through |W| the same way.
`_check(..., sensitive=True)` also proves on the test's own data that this bound rejects a kernel that is subtly wrong: mutated float64
references (one hidden unit's bias dropped, the first-layer activation skipped, the last K column ignored, sigmoid computed as tanh, two
outputs swapped) must each fall outside it.
"""

import math

import pytest
import torch
from torch import nn

from evotorch_b200 import _native as nat
from evotorch_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN = float("nan")
ACTS = ("none", "tanh", "relu", "sigmoid")
EPS32 = 2.0 ** -24
# C_ROUND, calibrated once on an H100 80GB HBM3: over every check in this file the largest |y - y64| / bound was 0.60 with C_ROUND = 2,
# at tail2 3-4-5 (a K of 3, where what 3xTF32 drops -- the lo x lo product, about 2^-22 of each term -- weighs most against K_eff); the
# next largest were 0.33 and 0.31, also at K <= 5, and 0.16 for the gather GEMM alone.  The data are seeded and the kernels
# deterministic, so this is a fixed margin; a larger C_ROUND would let the first-layer mutations of the 8-layer nets pass unseen
C_ROUND = 2.0
ACT_ERR = 1e-6

_F64 = {"none": lambda t: t, "tanh": torch.tanh, "relu": torch.relu, "sigmoid": torch.sigmoid}
MUTATIONS = ("bias_dropped", "act0_skipped", "last_k_ignored", "sigmoid_as_tanh", "outputs_swapped")


# ------------------------------------------------------------------------------------------------ float64 oracle
def _layers(P: torch.Tensor, dims, acts):
    """[(W (n, out, in), b (n, out), act)] in float64 from flat torch.nn.Linear-ordered parameter rows (W row-major, then b)."""
    n, off, out = P.shape[0], 0, []
    P = P.double()
    for l, act in enumerate(acts):
        W = P[:, off:off + dims[l] * dims[l + 1]].reshape(n, dims[l + 1], dims[l])
        off += dims[l] * dims[l + 1]
        out.append((W, P[:, off:off + dims[l + 1]], act))
        off += dims[l + 1]
    return out


def _input(x: torch.Tensor, n: int) -> torch.Tensor:
    """(n, B, in) float64: a shared batch (B, in) broadcast to every network, or per-network inputs (n, B, in) as they are."""
    x = x.double()
    return x.expand(n, *x.shape) if x.ndim == 2 else x


def _mutate(layers, mutation):
    if mutation is None:
        return layers
    layers = list(layers)
    W, b, act = layers[0]
    if mutation == "bias_dropped":  # per network, the first-layer unit whose bias moves the most
        j = b.abs().argmax(dim=1)
        b = b.clone()
        b[torch.arange(b.shape[0], device=b.device), j] = 0.0
    elif mutation == "act0_skipped":
        act = "none"
    elif mutation == "last_k_ignored":
        W = W.clone()
        W[..., -1] = 0.0
    layers[0] = (W, b, act)
    if mutation == "sigmoid_as_tanh":
        layers = [(W, b, "tanh" if a == "sigmoid" else a) for W, b, a in layers]
    return layers


def forward64(layers, x: torch.Tensor, mutation=None) -> torch.Tensor:
    """float64 forward -> (n, B, out); `mutation` (one of MUTATIONS) computes a subtly wrong variant instead."""
    layers = _mutate(layers, mutation)
    h = _input(x, layers[0][0].shape[0])
    for W, b, act in layers:
        h = torch.einsum("nbi,noi->nbo", h, W)
        if b is not None:
            h = h + b[:, None, :]
        h = _F64[act](h)
    if mutation == "outputs_swapped":  # output 0 and the output that differs from it the most
        j = int((h - h[..., :1]).abs().mean(dim=(0, 1)).argmax())
        order = list(range(h.shape[-1]))
        order[0], order[j] = j, 0
        h = h[..., order]
    return h


def bound64(layers, x: torch.Tensor, x_err: float = 0.0) -> torch.Tensor:
    """The per-element tolerance of the module docstring; `x_err` is a relative error of the input itself (the K8 normalisation)."""
    m = _input(x, layers[0][0].shape[0]).abs()
    e = m * x_err
    for W, b, act in layers:
        Wa = W.abs()
        m = torch.einsum("nbi,noi->nbo", m, Wa)
        e = torch.einsum("nbi,noi->nbo", e, Wa)
        if b is not None:
            m = m + b.abs()[:, None, :]
        if act in ("tanh", "sigmoid"):
            e = e + ACT_ERR
    k_eff = max(W.shape[2] for W, _, _ in layers)
    return C_ROUND * EPS32 * k_eff * m + e


def _within(y: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> bool:
    return bool(((y.double() - ref).abs() <= bound).all())  # NaN in y compares False


def _check(y: torch.Tensor, layers, x: torch.Tensor, sensitive: bool = False, x_err: float = 0.0) -> None:
    ref, bound = forward64(layers, x), bound64(layers, x, x_err)
    assert y.shape == ref.shape, (tuple(y.shape), tuple(ref.shape))
    err = (y.double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{bad.shape[0]} of {y.numel()} elements outside the bound; first at {i}: got {float(y[i])}, float64 "
                             f"{float(ref[i])}, bound {float(bound[i]):.3g}; worst |err| / bound {float((err / bound).max()):.3g}")
    if sensitive:
        acts = [a for _, _, a in layers]
        applicable = {"bias_dropped": layers[0][1] is not None, "act0_skipped": acts[0] != "none", "last_k_ignored": True,
                      "sigmoid_as_tanh": "sigmoid" in acts, "outputs_swapped": y.shape[-1] >= 2}
        for mutation in MUTATIONS:
            if applicable[mutation]:
                assert not _within(y, forward64(layers, x, mutation), bound), f"the bound does not reject `{mutation}`"


# ------------------------------------------------------------------------------------------------ data
def _population(n: int, dims, seed: int, pad: int = 0, offset: int = 0) -> torch.Tensor:
    """n flat parameter rows, weights ~ N(0, 1 / fan_in), biases ~ N(0, 0.25); with `pad` / `offset`, a view `offset` floats into rows
    of pitch L + pad + offset whose other elements are NaN."""
    g = torch.Generator().manual_seed(seed)  # drawn on the CPU: the same numbers on every machine
    parts = []
    for l in range(len(dims) - 1):
        parts.append(torch.randn(n, dims[l] * dims[l + 1], generator=g) / math.sqrt(dims[l]))
        parts.append(torch.randn(n, dims[l + 1], generator=g) * 0.5)
    P = torch.cat(parts, dim=1).to(DEV)
    if not pad and not offset:
        return P
    buf = torch.full((n, P.shape[1] + pad + offset), NAN, device=DEV)
    buf[:, offset:offset + P.shape[1]] = P
    return buf[:, offset:offset + P.shape[1]]


def _batch(B: int, K: int, seed: int) -> torch.Tensor:
    return torch.randn(B, K, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _rotated(n_layers: int, r: int):
    return tuple(ACTS[(l + r) % 4] for l in range(n_layers))


# ------------------------------------------------------------------------------------------------ ops.mlp_forward_shared, by branch
KS = (1, 2, 3, 4, 5, 31, 32, 33, 376)  # around the 32-wide K blocks and the 16-byte cut of a row's K axis
BS = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 257)  # around the 32-sample (generic tail) and 64-sample (tail2) passes, 128-col tiles
NS = (1, 2, 3, 7)  # N * h1 is not a multiple of the 128-row tile except at h1 = 128


def _og(dout: int) -> int:
    og = -(-dout // 4)
    return next(v for v in (1, 2, 4, 5, 8) if og <= v)


# mlp_tail2_kernel<OG>: two layers, dout <= 32, h1 % 4 == 0, h1 <= 508
TAIL2 = []
for _i, (_h1, _dout) in enumerate((h1, dout) for h1 in (4, 12, 128, 508) for dout in (1, 4, 5, 8, 9, 16, 17, 20, 21, 32)):
    TAIL2.append(pytest.param((KS[_i % 9], _h1, _dout), (ACTS[_i % 4], ACTS[(_i // 4) % 4]), NS[_i % 4], BS[_i % 12],
                              id=f"tail2_og{_og(_dout)}-{KS[_i % 9]}-{_h1}-{_dout}"))

# mlp_tail_kernel: 2-layer nets that tail2 does not take, and deep nets (every activation in every slot over the four rotations;
# a hidden width of 1 in each)
GENERIC = [
    ("generic2_dout33", (31, 40, 33), 0),  # dout > 32
    ("generic2_h1_30", (8, 30, 3), 1),  # h1 % 4 != 0
    ("generic2_h1_510", (33, 510, 9), 2),  # h1 % 4 != 0, wide
    ("generic2_h1_512", (5, 512, 2), 3),  # tail2 would need 205 952 B of shared memory
    ("generic2_h1_512_dout33", (376, 512, 33), 0),  # the widest two-layer net the generic tail stages: 202 884 B
] + [(f"generic4_r{r}", (k, 24, 1, 13, 6), r) for r, k in enumerate((1, 4, 376, 2))] \
  + [(f"generic8_r{r}", (k, 16, 1, 9, 24, 5, 12, 8, 3), r) for r, k in enumerate((3, 33, 31, 5))]
GENERIC = [pytest.param(dims, _rotated(len(dims) - 1, r), NS[j % 4], BS[(j + 5) % 12], id=tag) for j, (tag, dims, r) in enumerate(GENERIC)]


@pytest.mark.parametrize("dims,acts,n,B", TAIL2 + GENERIC)
def test_shared_forward_branch_matches_float64(dims, acts, n, B):
    seed = sum(dims) * 131 + n * 7 + B
    P, x = _population(n, dims, seed), _batch(B, dims[0], seed + 1)
    y = ops.mlp_forward_shared(P, x, dims, acts)
    _check(y, _layers(P, dims, acts), x, sensitive=True)


@pytest.mark.parametrize("dims,acts", [((5, 508, 7), ("tanh", "none")),  # tail2<2>
                                       ((5, 508, 20, 3), ("sigmoid", "relu", "tanh"))])  # generic tail
def test_shared_forward_multi_chunk(dims, acts):
    """h1 = 508, B = 4096: 2^30 / (508 * 4096 * 4) = 129 networks per chunk, so N = 300 runs as 129 + 129 + 42 (about 1 GiB of
    workspace).  Checked at every chunk's first and last network and at a few others."""
    n, B = 300, 4096
    P, x = _population(n, dims, 7), _batch(B, dims[0], 8)
    y = ops.mlp_forward_shared(P, x, dims, acts)
    g = torch.Generator().manual_seed(9)
    rows = sorted({0, 128, 129, 257, 258, 299} | set(torch.randint(0, n, (4,), generator=g).tolist()))
    idx = torch.tensor(rows, device=DEV)
    _check(y[idx], _layers(P[idx], dims, acts), x)


@pytest.mark.parametrize("dims,acts", [((37, 20, 6), ("sigmoid", "tanh")), ((37, 20, 9, 6), ("relu", "tanh", "sigmoid"))])
def test_shared_forward_padded_parameters_and_strided_batch(dims, acts):
    """Parameter rows 1-3 floats into NaN-padded rows of another pitch, and a batch that is a misaligned strided view."""
    n, B = 13, 70
    base = _population(n, dims, 21)
    wide = torch.full((B, dims[0] + 7), NAN, device=DEV)
    wide[:, 3:3 + dims[0]] = _batch(B, dims[0], 22)
    x = wide[:, 3:3 + dims[0]]
    for offset in (1, 2, 3):
        P = _population(n, dims, 21, pad=2, offset=offset)
        assert torch.equal(P, base) and P.stride(0) == base.shape[1] + 2 + offset
        y = ops.mlp_forward_shared(P, x, dims, acts)
        _check(y, _layers(P, dims, acts), x)


# ------------------------------------------------------------------------------------------------ the gather GEMM through the C ABI
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("with_bias", [True, False], ids=["bias", "no_bias"])
@pytest.mark.parametrize("kernel", ["one_tile", "persistent", "persistent_unit_fastest"])
def test_gather_gemm_c_abi(kernel, with_bias, act):
    """C[(i, h), b] = act(W_i[h, :] . X[b, :] + bias_i[h]) with bias 0 when bias_offset < 0.  Two shapes: M = 7 x 40 rows (not a
    multiple of the 128-row tile, a ragged K of 37) and 3 x 128 rows with K = 64 (the persistent kernel's 16-byte vector gather, rows
    at three misalignments).  Each into an aligned C with ldc % 4 == 0 (vector stores) and into a C one float off with an odd ldc
    (scalar stores); nothing outside C's logical extent is written."""
    lib, act_id = nat.lib(), ops.ACT_IDS[act]
    stream = torch.cuda.current_stream().cuda_stream
    for rpb, nb, K, n_cols in ((40, 7, 37, 70), (128, 3, 64, 130)):
        w_off = 3
        b_off = w_off + rpb * K
        L = (b_off + rpb + 2) | 1  # an odd row pitch
        g = torch.Generator().manual_seed(rpb * K + n_cols)
        P = torch.randn(nb, L, generator=g) / math.sqrt(K)
        P[:, b_off:b_off + rpb] *= 0.5 * math.sqrt(K)
        P, x = P.to(DEV), torch.randn(n_cols, K, generator=g).to(DEV)
        if kernel == "one_tile":  # TMA operand: 16-byte aligned rows
            X = torch.zeros(n_cols, (K + 3) // 4 * 4, device=DEV)
        else:  # any alignment
            X = torch.full((n_cols, K + 5), NAN, device=DEV)[:, 1:1 + K]
        X[:, :K] = x
        W = P[:, w_off:b_off].double().reshape(nb, rpb, K)
        layers = [(W, P[:, b_off:b_off + rpb].double() if with_bias else None, act)]
        M = nb * rpb
        for aligned in (True, False):
            ldc = (n_cols + 3) // 4 * 4 if aligned else n_cols + 1 + n_cols % 2
            skew = 0 if aligned else 1
            rows, cols = (nb * n_cols, rpb) if kernel == "persistent_unit_fastest" else (M, ldc)
            buf = torch.full((rows * cols + 8,), NAN, device=DEV)
            c_ptr = buf.data_ptr() + 4 * skew
            args = (P.data_ptr(), L, w_off, rpb, nb, X.data_ptr(), X.stride(0), n_cols, K, b_off if with_bias else -1, act_id, c_ptr, ldc)
            if kernel == "one_tile":
                rc = lib.evok_gemm_gather_rows(*args, stream)
            else:
                ws = torch.empty(lib.evok_gemm_gather_rows_workspace_bytes(n_cols, K), dtype=torch.uint8, device=DEV)
                rc = lib.evok_gemm_gather_rows_ws(*args, int(kernel == "persistent_unit_fastest"), ws.data_ptr(), ws.numel(), stream)
            nat.check(rc, kernel)
            torch.cuda.synchronize()
            C = buf[skew:skew + rows * cols].view(rows, cols)
            if kernel == "persistent_unit_fastest":  # C[(i * n_cols + b) * rpb + h]
                y, written = C.view(nb, n_cols, rpb), C
            else:  # C[(i * rpb + h) * ldc + b]
                y, written = C[:, :n_cols].reshape(nb, rpb, n_cols).transpose(1, 2), C[:, :n_cols]
            untouched = torch.ones_like(buf, dtype=torch.bool)
            untouched[skew:skew + rows * cols].view(rows, cols)[:, :written.shape[1]] = False
            assert bool(buf[untouched].isnan().all()), "a store outside C's logical extent"
            _check(y, layers, x, sensitive=True)


# ------------------------------------------------------------------------------------------------ Policy / NEProblem: nets the kernels cannot stage
def _sequential(dims, acts) -> nn.Sequential:
    mods = []
    for l, act in enumerate(acts):
        mods.append(nn.Linear(dims[l], dims[l + 1]))
        if act != "none":
            mods.append({"tanh": nn.Tanh, "relu": nn.ReLU, "sigmoid": nn.Sigmoid}[act]())
    return nn.Sequential(*mods)


# mlp_tail_kernel stages (2 * max_width * 33 + largest later layer's weights and bias) floats, at most 200 KB
@pytest.mark.parametrize("dims,acts,supported", [
    ((8, 256, 256, 2), ("tanh", "relu", "none"), False),  # 330 752 B
    ((8, 512, 40), ("tanh", "none"), False),  # 217 248 B
    ((8, 512, 34), ("relu", "sigmoid"), False),  # 204 936 B: the first dout past the limit at h1 = 512
    ((8, 512, 33), ("sigmoid", "none"), True),  # 202 884 B
    ((8, 196, 196, 2), ("tanh", "tanh", "none"), False),  # 206 192 B
    ((8, 195, 195, 2), ("tanh", "tanh", "none"), True),  # 204 360 B
], ids=lambda v: "-".join(map(str, v)) if isinstance(v, tuple) and isinstance(v[0], int) else None)
def test_policy_falls_back_for_nets_the_tail_cannot_stage(dims, acts, supported):
    from evotorch_b200.neuroevolution import NEProblem, Policy

    assert ops.mlp_forward_shared_supported(dims) == supported
    n, B = 5, 67
    P, x = _population(n, dims, sum(dims)), _batch(B, dims[0], 3)
    layers = _layers(P, dims, acts)
    net = _sequential(dims, acts)
    pol = Policy(net.to(DEV))
    before = ops.launch_count()
    y = pol.forward_shared(P, x)
    assert (ops.launch_count() > before) == supported  # the library kernels take exactly the nets the library says it supports
    _check(y, layers, x)
    prob = NEProblem("max", _sequential(dims, acts), lambda net: torch.zeros((), device=DEV), device=DEV)
    assert prob.solution_length == P.shape[1]
    _check(prob.batched_forward(P, x), layers, x)
    if not supported:
        with pytest.raises(ValueError, match="does not handle"):
            ops.mlp_forward_shared(P, x, dims, acts)


# ------------------------------------------------------------------------------------------------ K8: ops.mlp_forward at its limits
@pytest.mark.parametrize("n", [1, 2, 5])  # N = 1, 2: every row is an edge row (scalar loads); N = 5: the middle rows take float4 loads
@pytest.mark.parametrize("dims,acts", [
    ((1, 2048, 3, 17, 1, 40, 9, 33, 5), _rotated(8, 0)),  # 8 layers, a 2048-wide layer, a one-float input
    ((1, 2048, 3, 17, 1, 40, 9, 33, 5), _rotated(8, 2)),
    ((2048, 7, 2048, 2), ("sigmoid", "tanh", "relu")),
])
def test_per_policy_forward_at_its_limits(dims, acts, n):
    P = _population(n, dims, n + len(dims))
    x = _batch(n, dims[0], n)
    y = ops.mlp_forward(P, x, dims, acts)
    # (no mutation check here: with a fan-in of 2048 the bound is wider than the effect of one hidden unit's bias)
    _check(y[:, None, :], _layers(P, dims, acts), x[:, None, :])


@pytest.mark.parametrize("clip", [(None, 0.5), (-0.3, None)], ids=["hi_only", "lo_only"])
def test_per_policy_forward_prep_and_mask(clip):
    """`forward_prep`: x = clamp((obs - mean) / sqrt(max(sumsq / count - mean^2, min_variance)), lo, hi) with one side of the clip
    NaN (open) and min_variance in effect on a third of the features; `active` all false, then only the last row."""
    dims, acts = (12, 36, 4), ("tanh", "sigmoid")
    n, count, min_var = 9, 1000, 1e-2
    g = torch.Generator().manual_seed(5)
    mean = torch.randn(dims[0], generator=g)
    var = torch.rand(dims[0], generator=g) * 3 + 0.5
    var[::3] = 1e-4  # below min_variance: clamped
    obs_sum = (mean * count).to(DEV)
    obs_sumsq = ((var + mean * mean) * count).to(DEV)
    obs_count = torch.tensor([count], dtype=torch.int64, device=DEV)
    P = _population(n, dims, 6)
    obs = (torch.randn(n, dims[0], generator=g) * 2).to(DEV)
    m64 = obs_sum.double() / count
    v64 = torch.clamp(obs_sumsq.double() / count - m64 * m64, min=min_var)
    x64 = (obs.double() - m64) / v64.sqrt()
    x64 = torch.clamp(x64, min=clip[0], max=clip[1])
    kw = dict(obs_sum=obs_sum, obs_sumsq=obs_sumsq, obs_count=obs_count, min_variance=min_var, clip=clip)
    layers = _layers(P, dims, acts)
    y = ops.mlp_forward(P, obs, dims, acts, **kw)
    # the fp32 normalisation: a few roundings of each term, relative to |x| before the clip (the clip is 1-Lipschitz)
    _check(y[:, None, :], layers, x64[:, None, :], sensitive=True, x_err=16 * EPS32)
    for active in (torch.zeros(n, dtype=torch.bool, device=DEV), torch.arange(n, device=DEV) == n - 1):
        out = torch.full((n, dims[-1]), NAN, device=DEV)
        y = ops.mlp_forward(P, obs, dims, acts, out=out, active=active, **kw)
        assert y.data_ptr() == out.data_ptr()
        assert bool((y[~active] == 0).all())  # skipped policies get zero actions
        if bool(active.any()):
            idx = active.nonzero()[:, 0]
            _check(y[idx][:, None, :], _layers(P[idx], dims, acts), x64[idx][:, None, :], x_err=16 * EPS32)
