"""How the ranking (K3) and update (K5) entry points of the C ABI check their arguments and how many kernels each call launches.

The CPU part maps argument combinations to return codes; every case returns before a device is touched, so the launch count does
not move.  The GPU part pins the kernels one call launches on each path the size picks: the counting rank up to 8192 keys, the
self-scanning radix sort up to 256 tiles of 2048 keys (524 288 keys), the three-kernel radix sort above."""

import ctypes

import pytest

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build

NULLPTR, BADSIZE, BADENUM, WORKSPACE = -1, -2, -3, -4  # EVOK_E_* of include/evok.h
CENTERED, LINEAR, NES, NORMALIZED, RAW = 0, 1, 2, 3, 4
P = 64  # any non-null pointer: the argument checks never dereference it
BIG = 1 << 32  # N must fit the 32-bit sort indices


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def ws_bytes(lib, n):
    return lib.evok_rank_workspace_bytes(n)


def ptrs(*p):
    return (ctypes.c_void_p * len(p))(*p)


# Arguments that pass every check with nothing to do (N = 0 or no items), or, for the entry points that launch with any valid
# size, the smallest such size; each case changes some of them.
BASE = {
    "rank": dict(method=CENTERED, f=P, N=0, hib=0, w=P, perm=None, ws=P, ws_bytes=0),
    "argsort": dict(keys=P, N=0, desc=0, perm=P, ws=P, ws_bytes=0),
    "rank_table": dict(keys=P, N=0, desc=0, table=P, out=P, ws=P, ws_bytes=0),
    "elite_mask": dict(w=P, N=0, num_elites=0, mask=P, ws=P, ws_bytes=0),
    "weights_adjust": dict(w=P, N=0, mode=1),
    "rank_batched": dict(method=CENTERED, f=P, N=0, n_items=3, hib=0, w=P, ws=P, ws_bytes=0),
    "elite_mask_batched": dict(w=P, N=0, n_items=3, num_elites=0, mask=P, ws=P, ws_bytes=0),
    "weights_adjust_batched": dict(w=P, N=0, n_items=3, mode=1),
    "rank_sharded": dict(method=CENTERED, f=P, N=10, hib=0, world=2, rank=0, offsets=(0, 4, 10), keys=(P, P), fsum=(P, P), flags=(P, P),
                         epoch=P, done=P, err=P, w=P, mean=None, ws=P, ws_bytes=0),
    "clipup_step": dict(g=P, D=0, velocity=P, step_out=None, mu=None),
    "clipup_batched": dict(g=P, n_items=0, D=8, velocity=P, center=P, lr=P, mom=P, cap=P),
    "sigma_update": dict(sigma=P, g=P, D=0),
    "sigma_update_batched": dict(sigma=P, g=P, n_items=0, D=8, lr=P),
}


def call(lib, entry, a):
    if entry == "rank":
        return lib.evok_rank(a["method"], a["f"], a["N"], a["hib"], a["w"], a["perm"], a["ws"], a["ws_bytes"], None)
    if entry == "argsort":
        return lib.evok_argsort(a["keys"], a["N"], a["desc"], a["perm"], a["ws"], a["ws_bytes"], None)
    if entry == "rank_table":
        return lib.evok_rank_table(a["keys"], a["N"], a["desc"], a["table"], a["out"], a["ws"], a["ws_bytes"], None)
    if entry == "elite_mask":
        return lib.evok_elite_mask(a["w"], a["N"], a["num_elites"], a["mask"], a["ws"], a["ws_bytes"], None)
    if entry == "weights_adjust":
        return lib.evok_weights_adjust(a["w"], a["N"], a["mode"], None)
    if entry == "rank_batched":
        return lib.evok_rank_batched(a["method"], a["f"], a["N"], a["n_items"], a["hib"], a["w"], a["ws"], a["ws_bytes"], None)
    if entry == "elite_mask_batched":
        return lib.evok_elite_mask_batched(a["w"], a["N"], a["n_items"], a["num_elites"], a["mask"], a["ws"], a["ws_bytes"], None)
    if entry == "weights_adjust_batched":
        return lib.evok_weights_adjust_batched(a["w"], a["N"], a["n_items"], a["mode"], None)
    if entry == "rank_sharded":
        offs = None if a["offsets"] is None else (ctypes.c_int64 * len(a["offsets"]))(*a["offsets"])
        tables = [None if a[k] is None else ptrs(*a[k]) for k in ("keys", "fsum", "flags")]
        return lib.evok_rank_sharded(a["method"], a["f"], a["N"], a["hib"], a["world"], a["rank"], offs, *tables, a["epoch"], a["done"],
                                     a["err"], 10**9, a["w"], a["mean"], a["ws"], a["ws_bytes"], None)
    if entry == "clipup_step":
        return lib.evok_clipup_step(a["g"], a["D"], a["velocity"], 0.1, 0.9, 1.0, a["step_out"], a["mu"], None)
    if entry == "clipup_batched":
        return lib.evok_clipup_batched(a["g"], a["n_items"], a["D"], a["velocity"], a["center"], a["lr"], a["mom"], a["cap"], None)
    if entry == "sigma_update":
        return lib.evok_sigma_update(a["sigma"], a["g"], a["D"], 0.1, 0, None, float("nan"), None, float("nan"), None, float("nan"), None)
    return lib.evok_sigma_update_batched(a["sigma"], a["g"], a["n_items"], a["D"], a["lr"], 0, None, None, None, None)


def cases(lib):
    """(entry point, changed arguments, expected code)"""
    short = lambda n: ws_bytes(lib, n) - 1  # noqa: E731
    return [
        ("rank", {}, 0),
        ("rank", dict(f=None), NULLPTR),
        ("rank", dict(w=None), NULLPTR),
        ("rank", dict(ws=None), NULLPTR),
        ("rank", dict(method=-1), BADENUM),
        ("rank", dict(method=5), BADENUM),
        ("rank", dict(method=5, f=None), NULLPTR),
        ("rank", dict(method=5, N=-1), BADENUM),
        ("rank", dict(N=-1), BADSIZE),
        ("rank", dict(N=BIG), BADSIZE),
        ("rank", dict(N=BIG, ws=None), NULLPTR),
        ("rank", dict(N=BIG - 1), WORKSPACE),
        ("rank", dict(N=100, ws_bytes=short(100)), WORKSPACE),
        ("rank", dict(N=100, perm=P, ws_bytes=short(100)), WORKSPACE),
        ("rank", dict(N=9000, method=NES, ws_bytes=short(9000)), WORKSPACE),
        ("rank", dict(N=100, method=NORMALIZED, ws_bytes=short(100)), WORKSPACE),
        ("rank", dict(N=600000, method=RAW, perm=P, ws_bytes=short(600000)), WORKSPACE),
        ("rank", dict(method=RAW), 0),
        ("argsort", {}, 0),
        ("argsort", dict(keys=None), NULLPTR),
        ("argsort", dict(perm=None), NULLPTR),
        ("argsort", dict(ws=None, N=-1), NULLPTR),
        ("argsort", dict(N=-1), BADSIZE),
        ("argsort", dict(N=BIG), BADSIZE),
        ("argsort", dict(N=1, ws_bytes=short(1)), WORKSPACE),
        ("argsort", dict(N=8193, desc=1, ws_bytes=short(8193)), WORKSPACE),
        ("rank_table", {}, 0),
        ("rank_table", dict(keys=None), NULLPTR),
        ("rank_table", dict(table=None), NULLPTR),
        ("rank_table", dict(out=None), NULLPTR),
        ("rank_table", dict(ws=None), NULLPTR),
        ("rank_table", dict(N=-1), BADSIZE),
        ("rank_table", dict(N=BIG), BADSIZE),
        ("rank_table", dict(N=8192, ws_bytes=short(8192)), WORKSPACE),
        ("rank_table", dict(N=524289, ws_bytes=short(524289)), WORKSPACE),
        ("elite_mask", {}, 0),
        ("elite_mask", dict(w=None), NULLPTR),
        ("elite_mask", dict(mask=None), NULLPTR),
        ("elite_mask", dict(ws=None, num_elites=-1), NULLPTR),
        ("elite_mask", dict(N=-1), BADSIZE),
        ("elite_mask", dict(N=BIG, num_elites=1), BADSIZE),
        ("elite_mask", dict(num_elites=-1), BADSIZE),
        ("elite_mask", dict(num_elites=1), BADSIZE),
        ("elite_mask", dict(N=10, num_elites=11), BADSIZE),
        ("elite_mask", dict(N=10, num_elites=10, ws_bytes=short(10)), WORKSPACE),
        ("elite_mask", dict(N=20000, num_elites=0, ws_bytes=short(20000)), WORKSPACE),
        ("weights_adjust", {}, 0),
        ("weights_adjust", dict(w=None), NULLPTR),
        ("weights_adjust", dict(w=None, mode=0), NULLPTR),
        ("weights_adjust", dict(mode=0), BADENUM),
        ("weights_adjust", dict(mode=3), BADENUM),
        ("weights_adjust", dict(mode=0, N=-1), BADENUM),
        ("weights_adjust", dict(N=-1), BADSIZE),
        ("rank_batched", {}, 0),
        ("rank_batched", dict(N=100, n_items=0), 0),
        ("rank_batched", dict(f=None), NULLPTR),
        ("rank_batched", dict(w=None), NULLPTR),
        ("rank_batched", dict(ws=None), NULLPTR),
        ("rank_batched", dict(method=-1), BADENUM),
        ("rank_batched", dict(method=5, n_items=-1), BADENUM),
        ("rank_batched", dict(N=-1), BADSIZE),
        ("rank_batched", dict(N=BIG), BADSIZE),
        ("rank_batched", dict(n_items=-1), BADSIZE),
        ("rank_batched", dict(N=BIG - 1, n_items=1), WORKSPACE),
        ("rank_batched", dict(N=8193, ws_bytes=short(8193)), WORKSPACE),
        ("rank_batched", dict(N=8193, method=NES, ws_bytes=short(8193)), WORKSPACE),
        ("rank_batched", dict(N=100, method=NORMALIZED, ws_bytes=3 * 8 + 255), WORKSPACE),
        ("rank_batched", dict(N=100, method=RAW, n_items=70000, ws_bytes=65535 * 8 + 255), WORKSPACE),
        ("elite_mask_batched", {}, 0),
        ("elite_mask_batched", dict(N=100, n_items=0, num_elites=5), 0),
        ("elite_mask_batched", dict(w=None), NULLPTR),
        ("elite_mask_batched", dict(mask=None), NULLPTR),
        ("elite_mask_batched", dict(ws=None), NULLPTR),
        ("elite_mask_batched", dict(N=-1), BADSIZE),
        ("elite_mask_batched", dict(N=BIG), BADSIZE),
        ("elite_mask_batched", dict(n_items=-1), BADSIZE),
        ("elite_mask_batched", dict(num_elites=-1), BADSIZE),
        ("elite_mask_batched", dict(N=5, num_elites=6), BADSIZE),
        ("elite_mask_batched", dict(N=10000, num_elites=10, ws_bytes=short(10000)), WORKSPACE),
        ("weights_adjust_batched", {}, 0),
        ("weights_adjust_batched", dict(N=10, n_items=0), 0),
        ("weights_adjust_batched", dict(w=None), NULLPTR),
        ("weights_adjust_batched", dict(mode=2, w=None), NULLPTR),
        ("weights_adjust_batched", dict(mode=0), BADENUM),
        ("weights_adjust_batched", dict(mode=0, n_items=-1), BADENUM),
        ("weights_adjust_batched", dict(N=-1), BADSIZE),
        ("weights_adjust_batched", dict(n_items=-1), BADSIZE),
        ("rank_sharded", {}, WORKSPACE),
        ("rank_sharded", dict(offsets=None), NULLPTR),
        ("rank_sharded", dict(keys=None), NULLPTR),
        ("rank_sharded", dict(fsum=None), NULLPTR),
        ("rank_sharded", dict(flags=None), NULLPTR),
        ("rank_sharded", dict(epoch=None), NULLPTR),
        ("rank_sharded", dict(done=None), NULLPTR),
        ("rank_sharded", dict(err=None), NULLPTR),
        ("rank_sharded", dict(ws=None), NULLPTR),
        ("rank_sharded", dict(method=NORMALIZED), BADENUM),
        ("rank_sharded", dict(method=RAW), BADENUM),
        ("rank_sharded", dict(method=-1, world=0), BADENUM),
        ("rank_sharded", dict(world=0), BADSIZE),
        ("rank_sharded", dict(world=17), BADSIZE),
        ("rank_sharded", dict(rank=-1), BADSIZE),
        ("rank_sharded", dict(rank=2), BADSIZE),
        ("rank_sharded", dict(N=0, offsets=(0, 0, 0)), BADSIZE),
        ("rank_sharded", dict(N=BIG, offsets=(0, 4, BIG)), BADSIZE),
        ("rank_sharded", dict(offsets=(1, 4, 10)), BADSIZE),
        ("rank_sharded", dict(offsets=(0, 4, 9)), BADSIZE),
        ("rank_sharded", dict(offsets=(0, 11, 10)), BADSIZE),
        ("rank_sharded", dict(f=None), NULLPTR),
        ("rank_sharded", dict(w=None), NULLPTR),
        ("rank_sharded", dict(f=None, w=None, offsets=(0, 0, 10)), WORKSPACE),
        ("rank_sharded", dict(ws_bytes=short(4)), WORKSPACE),
        ("rank_sharded", dict(rank=1, ws_bytes=short(6)), WORKSPACE),
        ("rank_sharded", dict(ws_bytes=ws_bytes(lib, 4), keys=(P, None)), NULLPTR),
        ("rank_sharded", dict(ws_bytes=ws_bytes(lib, 4), flags=(None, P)), NULLPTR),
        ("clipup_step", {}, BADSIZE),
        ("clipup_step", dict(g=None), NULLPTR),
        ("clipup_step", dict(velocity=None, D=8), NULLPTR),
        ("clipup_step", dict(D=-1), BADSIZE),
        ("clipup_batched", {}, 0),
        ("clipup_batched", dict(g=None), NULLPTR),
        ("clipup_batched", dict(velocity=None), NULLPTR),
        ("clipup_batched", dict(center=None), NULLPTR),
        ("clipup_batched", dict(lr=None), NULLPTR),
        ("clipup_batched", dict(mom=None), NULLPTR),
        ("clipup_batched", dict(cap=None, D=0), NULLPTR),
        ("clipup_batched", dict(D=0), BADSIZE),
        ("clipup_batched", dict(n_items=-1), BADSIZE),
        ("sigma_update", {}, BADSIZE),
        ("sigma_update", dict(sigma=None), NULLPTR),
        ("sigma_update", dict(g=None, D=8), NULLPTR),
        ("sigma_update", dict(D=-3), BADSIZE),
        ("sigma_update_batched", {}, 0),
        ("sigma_update_batched", dict(sigma=None), NULLPTR),
        ("sigma_update_batched", dict(g=None), NULLPTR),
        ("sigma_update_batched", dict(lr=None, D=0), NULLPTR),
        ("sigma_update_batched", dict(D=0), BADSIZE),
        ("sigma_update_batched", dict(n_items=-1), BADSIZE),
    ]


def test_argument_checks_return_before_any_device_work(lib):
    launches = lib.evok_launch_count()
    failures = []
    for entry, change, want in cases(lib):
        got = call(lib, entry, {**BASE[entry], **change})
        if got != want:
            failures.append(f"{entry}({change}): {got}, expected {want}")
    assert not failures, "\n".join(failures)
    assert lib.evok_launch_count() == launches


# ------------------------------------------------------------------------------------------------ kernels launched per call
SIZES = (8192, 8193, 524288, 524289)  # counting | self-scanning radix, 256 tiles | 257 tiles, three-kernel radix


# (entry point, method or None) -> kernels one call launches at each of SIZES, recorded on the parent of the single ranking path.
# Counting rank: one launch for all items.  Radix sort: 8 launches up to 256 tiles, 13 above, then the scatter (+ the NES sum) per
# item.  The sharded ranking always sorts by radix, then pushes and merges.
EXPECTED = {
    ("rank", "centered"): (1, 9, 9, 14),
    ("rank", "nes"): (1, 10, 10, 15),
    ("rank", "normalized+perm"): (3, 11, 11, 16),  # mean / std + affine, then the argsort for perm
    ("rank", "normalized"): (2, 2, 2, 2),
    ("rank", "raw"): (1, 1, 1, 1),
    ("argsort", None): (1, 9, 9, 14),
    ("rank_table", None): (1, 9, 9, 14),
    ("elite_mask", None): (1, 9, 9, 14),
    ("rank_batched", "centered"): (1, 18, 18, 28),  # 2 items
    ("rank_batched", "nes"): (1, 20, 20, 30),
    ("rank_batched", "normalized"): (2, 2, 2, 2),
    ("elite_mask_batched", None): (1, 18, 18, 28),
    ("weights_adjust", None): (1, 1, 1, 1),
    ("weights_adjust_batched", None): (1, 1, 1, 1),
    ("rank_sharded", "centered"): (10, 10, 10, 15),
    ("rank_sharded", "nes"): (11, 11, 11, 16),
    ("clipup_step", None): (1, 1, 1, 1),  # K5: one launch, or one per 256 items (300 here)
    ("clipup_batched", None): (2, 2, 2, 2),
    ("sigma_update", None): (1, 1, 1, 1),
    ("sigma_update_batched", None): (2, 2, 2, 2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_launches_per_call(lib, n):
    import torch

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(n)
    f = torch.round(torch.randn(2, n, device=dev, generator=g) * 20) / 20
    ws = torch.empty(max(ws_bytes(lib, n), 8 * 2 + 256), dtype=torch.uint8, device=dev)
    out = torch.empty(2, n, device=dev)
    perm = torch.empty(n, dtype=torch.int64, device=dev)
    table = torch.randn(n, device=dev, generator=g)
    st = torch.cuda.current_stream().cuda_stream
    W = (ws.data_ptr(), ws.numel(), st)
    f0, o0 = f[0].data_ptr(), out.data_ptr()
    # world-1 sharded ranking: this rank's buffers are its own peer table
    keys, fsum = torch.zeros(n, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.float64, device=dev)
    flags, epoch = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
    done, err, mean = torch.zeros(4, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, device=dev)
    offs = (ctypes.c_int64 * 2)(0, n)
    items, D = 300, 64
    gk = torch.randn(items, D, device=dev, generator=g)
    vel, cen = torch.zeros(items, D, device=dev), torch.ones(items, D, device=dev)
    hp = (ctypes.c_float * items)(*[0.1] * items)
    nan = float("nan")

    def sharded(method):
        return lambda: lib.evok_rank_sharded(method, f0, n, 0, 1, 0, offs, ptrs(keys.data_ptr()), ptrs(fsum.data_ptr()), ptrs(flags.data_ptr()),
                                             epoch.data_ptr(), done.data_ptr(), err.data_ptr(), int(5e9), o0, mean.data_ptr(), *W)

    calls = {
        ("rank", "centered"): lambda: lib.evok_rank(CENTERED, f0, n, 0, o0, perm.data_ptr(), *W),
        ("rank", "nes"): lambda: lib.evok_rank(NES, f0, n, 1, o0, None, *W),
        ("rank", "normalized+perm"): lambda: lib.evok_rank(NORMALIZED, f0, n, 0, o0, perm.data_ptr(), *W),
        ("rank", "normalized"): lambda: lib.evok_rank(NORMALIZED, f0, n, 0, o0, None, *W),
        ("rank", "raw"): lambda: lib.evok_rank(RAW, f0, n, 1, o0, None, *W),
        ("argsort", None): lambda: lib.evok_argsort(f0, n, 1, perm.data_ptr(), *W),
        ("rank_table", None): lambda: lib.evok_rank_table(f0, n, 0, table.data_ptr(), o0, *W),
        ("elite_mask", None): lambda: lib.evok_elite_mask(f0, n, n // 4, o0, *W),
        ("rank_batched", "centered"): lambda: lib.evok_rank_batched(CENTERED, f0, n, 2, 0, o0, *W),
        ("rank_batched", "nes"): lambda: lib.evok_rank_batched(NES, f0, n, 2, 1, o0, *W),
        ("rank_batched", "normalized"): lambda: lib.evok_rank_batched(NORMALIZED, f0, n, 2, 0, o0, *W),
        ("elite_mask_batched", None): lambda: lib.evok_elite_mask_batched(f0, n, 2, n // 4, o0, *W),
        ("weights_adjust", None): lambda: lib.evok_weights_adjust(o0, n, 1, st),
        ("weights_adjust_batched", None): lambda: lib.evok_weights_adjust_batched(o0, n, 2, 2, st),
        ("rank_sharded", "centered"): sharded(CENTERED),
        ("rank_sharded", "nes"): sharded(NES),
        ("clipup_step", None): lambda: lib.evok_clipup_step(gk.data_ptr(), D, vel.data_ptr(), 0.1, 0.9, 1.0, None, cen.data_ptr(), st),
        ("clipup_batched", None): lambda: lib.evok_clipup_batched(gk.data_ptr(), items, D, vel.data_ptr(), cen.data_ptr(), hp, hp, hp, st),
        ("sigma_update", None): lambda: lib.evok_sigma_update(cen.data_ptr(), gk.data_ptr(), D, 0.1, 0, None, nan, None, nan, None, nan, st),
        ("sigma_update_batched", None): lambda: lib.evok_sigma_update_batched(cen.data_ptr(), gk.data_ptr(), items, D, hp, 0, None, None, None, st),
    }
    got, want = {}, {}
    for (entry, method), run in calls.items():
        before = lib.evok_launch_count()
        assert run() == 0, (entry, method)
        got[(entry, method)] = lib.evok_launch_count() - before
        want[(entry, method)] = EXPECTED[(entry, method)][SIZES.index(n)]
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    assert got == want


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["transposed", "float64", "cpu"])
def test_batched_wrappers_refuse_what_the_kernels_cannot_read(layout):
    import torch

    from evotorch_b200 import ops

    w = {"transposed": torch.randn(64, 3, device="cuda").t(), "float64": torch.randn(3, 64, device="cuda", dtype=torch.float64),
         "cpu": torch.randn(3, 64)}[layout]
    with pytest.raises(ValueError, match="weights: expected a contiguous float32 CUDA tensor of shape"):
        ops.weights_adjust_batched_(w, 1)
    with pytest.raises(ValueError, match="weights: expected a contiguous float32 CUDA tensor of shape"):
        ops.elite_mask_batched(w, 8)
