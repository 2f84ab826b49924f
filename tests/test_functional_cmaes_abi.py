"""The batched entry points of the functional CMA-ES without a device: return codes of evok_gemm_nt_batched,
evok_gemm_nt_affine_batched, evok_transpose_pair_batched, evok_rank_table_batched, evok_cmaes_row_weights_batched and
evok_cmaes_vector_update_batched on calls that return before any device work (nothing is launched), the workspace that
evok_gemm_nt_batched_workspace_bytes asks for, and CPU checks of the float64 references the GPU tests rely on: the stable
ranking, and the mutated generations that the whole-generation bound has to reject."""

import numpy as np
import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build
from evotorch_b200.algorithms.functional import cmaes
from evotorch_b200.algorithms.functional.funccmaes import _assigned_weights
from oracle import functional_cmaes_oracle as FO

NULLPTR, BADSIZE, WORKSPACE = -1, -2, -4  # EVOK_E_* of include/evok.h
P = 64  # any non-null, 16-byte aligned pointer: the argument checks never dereference it
U = 68  # not 16-byte aligned


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def _no_launch(lib, call):
    before = lib.evok_launch_count()
    rc = call()
    assert lib.evok_launch_count() == before
    return rc


# M = N = 4, K = 8: 2 items of A / B at item stride 32 (aligned), C at 16; with ws_bytes = 0 a valid call stops at EVOK_E_WORKSPACE
GEMM_BASE = dict(A=P, lda=8, sa=32, B=P, ldb=8, sb=32, items=2, M=4, N=4, K=8, C=P, ldc=4, sc=16, C2=None, ldc2=0, sc2=0, alpha=None, salpha=0,
                 bias=None, sbias=0, ws=P, ws_bytes=0)
GEMM_CASES = [
    ({}, WORKSPACE),
    (dict(items=0), 0),
    (dict(items=-1), BADSIZE),
    (dict(A=None), NULLPTR),
    (dict(B=None), NULLPTR),
    (dict(C=None), NULLPTR),
    (dict(ws=None), NULLPTR),
    (dict(A=None, items=0), NULLPTR),
    (dict(sa=-32), BADSIZE),
    (dict(sb=-32), BADSIZE),
    (dict(sa=-32, items=0), BADSIZE),
    (dict(lda=7), BADSIZE),
    (dict(ldb=7), BADSIZE),
    (dict(ldc=3), BADSIZE),
    (dict(M=0), BADSIZE),
    (dict(K=0), BADSIZE),
    (dict(K=2**31, lda=2**31, ldb=2**31), BADSIZE),
    (dict(sc=15), BADSIZE),  # item b's last row overlaps item b+1's first
    (dict(sc=15, items=1), WORKSPACE),  # one item: no overlap is possible
    (dict(sc=0), BADSIZE),
    (dict(C2=P, ldc2=4, sc2=16), WORKSPACE),
    (dict(C2=P, ldc2=4, sc2=15), BADSIZE),
    (dict(C2=P, ldc2=3, sc2=16), BADSIZE),
    (dict(C2=P, ldc2=4, sc2=0, items=1), WORKSPACE),
    (dict(alpha=P, salpha=-1), BADSIZE),
    (dict(bias=P, sbias=-4), BADSIZE),
    (dict(A=U), WORKSPACE),  # the split copies need a workspace too
]


def gemm_call(lib, a):
    return lib.evok_gemm_nt_batched(a["A"], a["lda"], a["sa"], a["B"], a["ldb"], a["sb"], a["items"], a["M"], a["N"], a["K"], a["C"], a["ldc"], a["sc"],
                                    a["C2"], a["ldc2"], a["sc2"], a["alpha"], a["salpha"], a["bias"], a["sbias"], a["ws"], a["ws_bytes"], None)


@pytest.mark.parametrize("changes,code", GEMM_CASES)
def test_gemm_nt_batched_codes(lib, changes, code):
    assert _no_launch(lib, lambda: gemm_call(lib, dict(GEMM_BASE, **changes))) == code


AFFINE_BASE = dict(GEMM_BASE, k=P, sk=3, E=None, lde=0, se=0, u=None, su=0)
AFFINE_CASES = [
    ({}, WORKSPACE),
    (dict(items=0), 0),
    (dict(k=None), NULLPTR),
    (dict(k=None, items=0), NULLPTR),
    (dict(A=None), NULLPTR),
    (dict(sk=-3), BADSIZE),
    (dict(sk=0), WORKSPACE),  # one k shared by every item
    (dict(E=P, lde=4, se=16), WORKSPACE),
    (dict(E=P, lde=4, se=0), WORKSPACE),  # one E shared by every item
    (dict(E=P, lde=3, se=16), BADSIZE),  # lde < N
    (dict(E=P, lde=4, se=-16), BADSIZE),
    (dict(u=P, su=4), WORKSPACE),
    (dict(u=P, su=0), WORKSPACE),
    (dict(u=P, su=-4), BADSIZE),
    (dict(u=P, su=4, N=3), BADSIZE),  # u needs M == N
    (dict(u=None, N=3, sc=16), WORKSPACE),
    (dict(sc=15), BADSIZE),
    (dict(sc=15, items=1), WORKSPACE),
    (dict(lda=7), BADSIZE),
    (dict(sa=-32), BADSIZE),
]


def affine_call(lib, a):
    return lib.evok_gemm_nt_affine_batched(a["A"], a["lda"], a["sa"], a["B"], a["ldb"], a["sb"], a["items"], a["M"], a["N"], a["K"], a["C"], a["ldc"],
                                           a["sc"], a["k"], a["sk"], a["E"], a["lde"], a["se"], a["u"], a["su"], a["ws"], a["ws_bytes"], None)


@pytest.mark.parametrize("changes,code", AFFINE_CASES)
def test_gemm_nt_affine_batched_codes(lib, changes, code):
    assert _no_launch(lib, lambda: affine_call(lib, dict(AFFINE_BASE, **changes))) == code


# rows (popsize) 40 and cols (D) 8: out_w / out_p [item][col][row] at pitch ldo = 40, item stride 320
TRANSPOSE_BASE = dict(inp=P, ldi=8, si=320, rows=40, cols=8, w=P, sw=40, out_w=P, out_p=P, ldo=40, so=320, items=0)
TRANSPOSE_CASES = [
    ({}, 0),
    (dict(inp=None), NULLPTR),
    (dict(w=None), NULLPTR),
    (dict(out_w=None), NULLPTR),
    (dict(out_p=None), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(rows=0), BADSIZE),
    (dict(cols=0), BADSIZE),
    (dict(ldi=7), BADSIZE),
    (dict(ldo=39), BADSIZE),
    (dict(si=-320), BADSIZE),
    (dict(sw=-40), BADSIZE),
    (dict(so=319, items=2), BADSIZE),  # item b's out_w / out_p overlap item b+1's
    (dict(so=0, items=2), BADSIZE),
    (dict(rows=65535 * 32 + 1, ldo=65535 * 32 + 1, so=8 * (65535 * 32 + 1), items=1), BADSIZE),  # more than 65535 row tiles
]


def transpose_call(lib, a):
    return lib.evok_transpose_pair_batched(a["inp"], a["ldi"], a["si"], a["rows"], a["cols"], a["w"], a["sw"], a["out_w"], a["out_p"], a["ldo"], a["so"],
                                           a["items"], None)


@pytest.mark.parametrize("changes,code", TRANSPOSE_CASES)
def test_transpose_pair_batched_codes(lib, changes, code):
    assert _no_launch(lib, lambda: transpose_call(lib, dict(TRANSPOSE_BASE, **changes))) == code


RANK_BASE = dict(keys=P, N=16, items=0, table=P, out=P, ws=P, ws_bytes=0)
RANK_CASES = [
    ({}, 0),
    (dict(N=0, items=3), 0),
    (dict(keys=None), NULLPTR),
    (dict(table=None), NULLPTR),
    (dict(out=None), NULLPTR),
    (dict(ws=None), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(N=-1), BADSIZE),
    (dict(N=2**32), BADSIZE),
    (dict(N=2**32, items=0), BADSIZE),
    (dict(N=2**32 - 1), 0),  # a valid size; no items: nothing to do
]


@pytest.mark.parametrize("changes,code", RANK_CASES)
def test_rank_table_batched_codes(lib, changes, code):
    a = dict(RANK_BASE, **changes)
    rc = _no_launch(lib, lambda: lib.evok_rank_table_batched(a["keys"], a["N"], a["items"], 1, a["table"], a["out"], a["ws"], a["ws_bytes"], None))
    assert rc == code


ROW_BASE = dict(aw=P, Z=P, sz=32, ldz=8, items=0, N=4, D=8, w_pos=P, w_act=P)
ROW_CASES = [
    ({}, 0),
    (dict(aw=None), NULLPTR),
    (dict(Z=None), NULLPTR),
    (dict(w_pos=None), NULLPTR),
    (dict(w_act=None), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(N=0), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(ldz=7), BADSIZE),  # ldz < D
    (dict(sz=-32), BADSIZE),
    (dict(sz=-32, items=2), BADSIZE),
]


@pytest.mark.parametrize("changes,code", ROW_CASES)
def test_cmaes_row_weights_batched_codes(lib, changes, code):
    a = dict(ROW_BASE, **changes)
    rc = _no_launch(lib, lambda: lib.evok_cmaes_row_weights_batched(a["aw"], a["Z"], a["sz"], a["ldz"], a["items"], a["N"], a["D"], 1, a["w_pos"],
                                                                    a["w_act"], None))
    assert rc == code


VEC_BASE = dict(local=P, shaped=P, items=0, D=8, m=P, ps=P, pc=P, sigma=P, consts=True, k=P)
VEC_CASES = [
    ({}, 0),
    (dict(local=None), NULLPTR),
    (dict(shaped=None), NULLPTR),
    (dict(m=None), NULLPTR),
    (dict(ps=None), NULLPTR),
    (dict(pc=None), NULLPTR),
    (dict(sigma=None), NULLPTR),
    (dict(consts=None), NULLPTR),
    (dict(k=None), NULLPTR),
    (dict(items=-1), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(D=0, items=0), BADSIZE),
]


@pytest.mark.parametrize("changes,code", VEC_CASES)
def test_cmaes_vector_update_batched_codes(lib, changes, code):
    import ctypes

    a = dict(VEC_BASE, **changes)
    consts = (ctypes.c_float * 10)(*([0.5] * 10)) if a["consts"] else None
    rc = _no_launch(lib, lambda: lib.evok_cmaes_vector_update_batched(a["local"], a["shaped"], a["items"], a["D"], a["m"], a["ps"], a["pc"], a["sigma"],
                                                                      3, consts, 0, a["k"], None))
    assert rc == code


def _al(x):
    return (x + 1023) // 1024 * 1024


@pytest.mark.parametrize("items", [1, 3, 65535, 65536, 70000])
@pytest.mark.parametrize("M,N,K", [(4, 4, 8), (5, 3, 7), (130, 129, 33)])
def test_gemm_batched_workspace_follows_the_plan(lib, items, M, N, K):
    """1024 bytes (alignment slack only) when both operands are read by the GEMM itself; otherwise hi / lo copies of both, sized to
    min(items, 65535) items per per-item operand and to one copy of a shared one."""
    ws = lib.evok_gemm_nt_batched_workspace_bytes
    ldk = (K + 3) // 4 * 4
    chunk = min(items, 65535)
    lda = ldk  # a pitch that is a multiple of 4 floats
    aligned = dict(sa=M * lda, sb=N * lda)

    def split(per_a, per_b):
        a = _al((chunk if per_a else 1) * M * ldk * 4)
        b = _al((chunk if per_b else 1) * N * ldk * 4)
        return 2 * a + 2 * b + 1024

    assert ws(P, lda, aligned["sa"], P, lda, aligned["sb"], items, M, N, K) == 1024
    assert ws(P, lda, 0, P, lda, 0, items, M, N, K) == 1024
    assert ws(P, lda, aligned["sa"], P, lda, 0, items, M, N, K) == 1024
    # an unaligned base, pitch or item stride of either operand sends both through the split copies
    assert ws(U, lda, aligned["sa"], P, lda, aligned["sb"], items, M, N, K) == split(True, True)
    assert ws(P, lda, aligned["sa"], U, lda, aligned["sb"], items, M, N, K) == split(True, True)
    assert ws(P, lda, aligned["sa"] + 2, P, lda, aligned["sb"], items, M, N, K) == split(True, True)
    assert ws(P, K + 1 if (K + 1) % 4 else K + 2, 0, P, lda, aligned["sb"], items, M, N, K) == split(False, True)
    assert ws(P, lda, aligned["sa"], U, lda, 0, items, M, N, K) == split(True, False)  # per-item aligned A, shared unaligned B
    assert ws(U, lda, 0, U, lda, 0, items, M, N, K) == split(False, False)
    # items that overlap cannot be one plane each of a rank-3 map
    assert ws(P, lda, aligned["sa"] - 4, P, lda, aligned["sb"], items, M, N, K) == split(True, True)


@pytest.mark.parametrize("items,M,N,K", [(0, 4, 4, 8), (-1, 4, 4, 8), (3, 0, 4, 8), (3, 4, 4, 0)])
def test_gemm_batched_workspace_of_empty_products(lib, items, M, N, K):
    assert lib.evok_gemm_nt_batched_workspace_bytes(U, K, 0, U, K, 0, items, M, N, K) == 1024


# ------------------------------------------------------------------------------------------------ the references themselves
def _keys(rng, items, n):
    """Fitnesses with ties inside and across items, +-0, +-inf and NaN."""
    k = rng.integers(-3, 4, size=(items, n)).astype(np.float32)
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], dtype=np.float32)
    mask = rng.random((items, n)) < 0.3
    k[mask] = rng.choice(special, size=int(mask.sum()))
    if items > 1:
        k[1] = k[0]
    return k


@pytest.mark.parametrize("n", [1, 2, 7, 40, 1025])
@pytest.mark.parametrize("maximize", [False, True])
def test_stable_rank_reference_matches_the_torch_path(n, maximize):
    """The GPU tests' ranking reference and the CPU tell's argsort / scatter assign the same weight to every row, bit for bit."""
    rng = np.random.default_rng(n + 7 * maximize)
    keys = _keys(rng, 5, n)
    table = rng.standard_normal(n).astype(np.float32)
    ref = FO.stable_rank_table(keys, maximize, table)
    got = _assigned_weights(torch.from_numpy(keys), maximize, torch.from_numpy(table)).numpy()
    assert np.array_equal(ref.view(np.int32), got.view(np.int32))


def test_nan_ranks_as_the_largest_value():
    keys = np.array([[1.0, np.nan, np.inf, -np.inf, -0.0, 0.0]], dtype=np.float32)
    table = np.arange(6, dtype=np.float32)
    # descending ("max"): NaN first (best), then +inf, 1, then -0 / +0 in index order, -inf last
    assert FO.stable_rank_table(keys, True, table).tolist() == [[2, 0, 1, 5, 3, 4]]
    # ascending ("min"): -inf first, -0 / +0 in index order, 1, +inf, NaN last (worst)
    assert FO.stable_rank_table(keys, False, table).tolist() == [[3, 5, 4, 0, 1, 2]]


def _linear(x):
    return x.sum(-1)


def _cpu_case(kind):
    """A CPU float32 state and one asked population on which `kind`'s mutation must change the reference."""
    torch.manual_seed(5)
    items, d = 3, 6
    kw = dict(stdev_min=0.44, stdev_max=0.46) if kind == "clamp" else {}
    state = cmaes(center_init=torch.randn(items, d), stdev_init=0.45 if kind == "clamp" else 1.0, objective_sense="max" if kind == "max" else "min",
                  **kw)
    if kind == "h0":
        # ||p_sigma|| far above the h_sig threshold, and a p_c for the rank-1 term to carry
        state = state._replace(p_sigma=torch.full((items, d), 5.0), p_c=torch.full((items, d), 2.0))
    x = torch.randn(items, state.popsize, d) * state.sigma[:, None, None] + state.center[:, None, :]
    f = _linear(x)
    return state, x, f


MUTATION_CASES = {"sense_flipped": "max", "neighbour_fitness": "min", "neighbour_rows": "min", "h_sig_one": "h0", "m_new_sigma": "h0",
                  "csa_swapped": "min", "no_active": "min", "k2_no_wpc": "h0", "clamp_old_sigma": "clamp"}


@pytest.mark.parametrize("mutation", FO.MUTATIONS)
def test_every_mutated_reference_differs_from_the_true_one(mutation):
    """On the CPU case meant to catch it, each mutated reference moves the new state far outside the bound (measured against the
    true reference standing in for the kernels' result)."""
    from evotorch_b200.algorithms.functional import cmaes_tell

    assert set(MUTATION_CASES) == set(FO.MUTATIONS)
    state, x, f = _cpu_case(MUTATION_CASES[mutation])
    new = cmaes_tell(state, x, f)  # the CPU path: the same algorithm in float32
    rec = []
    assert max(FO.tell_bound(state, x, f, new, record=rec)) <= 1.0
    if mutation in ("h_sig_one", "m_new_sigma", "k2_no_wpc"):
        assert all(r["h"] == 0.0 for r in rec)
    if mutation == "clamp_old_sigma":
        assert any(((r["stdevs"] < 0.44) | (r["stdevs"] > 0.46)).any() for r in rec)
    assert min(FO.tell_bound(state, x, f, new, mutation=mutation)) > 1.0
