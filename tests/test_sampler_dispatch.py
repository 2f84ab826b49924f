"""How the four objective entry points of the C ABI (evok_sample_eval, _sq, _push, evok_eval) check their arguments and which
kernel they launch, for the built-in objectives and for one registered at run time.

The CPU part maps argument combinations to return codes; every case returns before a device is touched, so the launch count
does not move.  The GPU part launches each entry point under torch.profiler and reads the kernel's template arguments and block
size from the trace: the bit-comparison tests give the same numbers for a vectorised or scalar, stored or lazy kernel, so they
would not notice a wrong choice."""

import ctypes
import json
import re

import pytest

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build

NULLPTR, BADSIZE, BADENUM, ODDROWS = -1, -2, -3, -5  # EVOK_E_* of include/evok.h
USER_BASE, USER_CAPACITY, MAX_PEERS = 64, 256, 16
KERNEL_NAMES = 22
P = 64  # any non-null pointer: the argument checks never dereference it


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


@pytest.fixture(scope="module")
def registered(lib):
    """The id of an objective registered from a dummy image (registration stores it; nothing here loads it)."""
    img = b"\x7fELF" + bytes(60)
    names = (ctypes.c_char_p * KERNEL_NAMES)(*[b"k"] * KERNEL_NAMES)
    out = ctypes.c_int(-1)
    assert lib.evok_objective_register(img, len(img), names, KERNEL_NAMES, ctypes.byref(out)) == 0
    return out.value


def peers(*ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


# Arguments that pass every check: n_rows = 0, so the three entry points that return early for no rows do so.  _push launches
# even without rows, so each of its cases breaks one argument.
BASE = {
    "sample_eval": dict(X=P, ldx=8, mu=P, sigma=P, row0=0, n_rows=0, D=8, sym=1, f=P),
    "sample_eval_sq": dict(X=P, ldx=8, mu=P, sigma=P, row0=0, n_rows=0, D=8, f=P, q=P),
    "sample_eval_push": dict(X=P, ldx=8, mu=P, sigma=P, row0=0, n_rows=0, D=8, sym=1, world=2, rank=1, peer_f=(P, P),
                             peer_flags=(P, P), epoch=P, done=P),
    "evaluate": dict(X=P, ldx=8, n_rows=0, D=8, f=P),
}


def call(lib, entry, objective, a):
    if entry == "sample_eval":
        return lib.evok_sample_eval(objective, a["X"], a["ldx"], a["mu"], a["sigma"], a["row0"], a["n_rows"], a["D"], a["sym"], 0, 0,
                                    None, a["f"], None)
    if entry == "sample_eval_sq":
        return lib.evok_sample_eval_sq(objective, a["X"], a["ldx"], a["mu"], a["sigma"], a["row0"], a["n_rows"], a["D"], 0, 0, None,
                                       a["f"], a["q"], None)
    if entry == "sample_eval_push":
        pf = None if a["peer_f"] is None else peers(*a["peer_f"])
        pg = None if a["peer_flags"] is None else peers(*a["peer_flags"])
        return lib.evok_sample_eval_push(objective, a["X"], a["ldx"], a["mu"], a["sigma"], a["row0"], a["n_rows"], a["D"], a["sym"], 0,
                                         0, None, a["world"], a["rank"], pf, pg, a["epoch"], a["done"], None)
    return lib.evok_eval(objective, a["X"], a["ldx"], a["n_rows"], a["D"], a["f"], None)


# (entry point, changed arguments, expected code for EVOK_OBJ_NONE, for a fused objective (built-in 1-3 or registered), for an
# id that names no objective)
CASES = [
    ("sample_eval", {}, 0, 0, BADENUM),
    ("sample_eval", dict(mu=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval", dict(sigma=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval", dict(X=None), NULLPTR, 0, BADENUM),
    ("sample_eval", dict(f=None), 0, NULLPTR, BADENUM),
    ("sample_eval", dict(X=None, f=None), NULLPTR, NULLPTR, BADENUM),
    ("sample_eval", dict(X=None, n_rows=-2), NULLPTR, BADSIZE, BADENUM),
    ("sample_eval", dict(f=None, D=0), BADSIZE, NULLPTR, BADENUM),
    ("sample_eval", dict(n_rows=-2), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(n_rows=-1), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(D=0), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(D=-4), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(row0=-2), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(ldx=7), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(ldx=7, X=None), NULLPTR, 0, BADENUM),
    ("sample_eval", dict(ldx=7, sym=0), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(n_rows=6, D=0), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(n_rows=3), ODDROWS, ODDROWS, BADENUM),
    ("sample_eval", dict(row0=1), ODDROWS, ODDROWS, BADENUM),
    ("sample_eval", dict(row0=1, ldx=7), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(row0=1, sym=0), 0, 0, BADENUM),
    ("sample_eval", dict(n_rows=3, sym=0, D=0), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval", dict(n_rows=3, mu=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_sq", {}, 0, 0, BADENUM),
    ("sample_eval_sq", dict(mu=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_sq", dict(sigma=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_sq", dict(q=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_sq", dict(q=None, D=0), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_sq", dict(X=None), NULLPTR, 0, BADENUM),
    ("sample_eval_sq", dict(f=None), 0, NULLPTR, BADENUM),
    ("sample_eval_sq", dict(X=None, D=0), NULLPTR, BADSIZE, BADENUM),
    ("sample_eval_sq", dict(f=None, n_rows=-1), BADSIZE, NULLPTR, BADENUM),
    ("sample_eval_sq", dict(n_rows=-1), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval_sq", dict(D=0), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval_sq", dict(row0=-1), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval_sq", dict(ldx=7), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval_sq", dict(ldx=7, X=None), NULLPTR, 0, BADENUM),
    ("sample_eval_sq", dict(row0=1), 0, 0, BADENUM),  # not symmetric: any first row
    ("sample_eval_sq", dict(row0=3, n_rows=-3), BADSIZE, BADSIZE, BADENUM),
    ("sample_eval_push", dict(mu=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(sigma=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(peer_f=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(peer_flags=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(epoch=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(done=None), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(done=None, world=0), NULLPTR, NULLPTR, NULLPTR),
    ("sample_eval_push", dict(world=0), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(world=MAX_PEERS + 1), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(rank=-1), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(rank=2), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(rank=2, n_rows=3), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(n_rows=-2), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(D=0), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(row0=-2), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(ldx=7), BADENUM, BADSIZE, BADENUM),
    ("sample_eval_push", dict(n_rows=3), BADENUM, ODDROWS, BADENUM),
    ("sample_eval_push", dict(row0=1), BADENUM, ODDROWS, BADENUM),
    ("sample_eval_push", dict(n_rows=3, peer_f=(P, None)), BADENUM, ODDROWS, BADENUM),
    ("sample_eval_push", dict(peer_f=(P, None)), BADENUM, NULLPTR, BADENUM),
    ("sample_eval_push", dict(peer_flags=(None, P)), BADENUM, NULLPTR, BADENUM),
    ("sample_eval_push", dict(peer_f=(P, None), X=None, ldx=7, sym=0, row0=1, n_rows=5), BADENUM, NULLPTR, BADENUM),
    ("sample_eval_push", dict(world=1, rank=0, peer_f=(None,)), BADENUM, NULLPTR, BADENUM),
    ("evaluate", {}, BADENUM, 0, BADENUM),
    ("evaluate", dict(X=None), NULLPTR, NULLPTR, NULLPTR),
    ("evaluate", dict(f=None), NULLPTR, NULLPTR, NULLPTR),
    ("evaluate", dict(f=None, D=0), NULLPTR, NULLPTR, NULLPTR),
    ("evaluate", dict(n_rows=-1), BADENUM, BADSIZE, BADENUM),
    ("evaluate", dict(D=0), BADENUM, BADSIZE, BADENUM),
    ("evaluate", dict(ldx=7), BADENUM, BADSIZE, BADENUM),
    ("evaluate", dict(ldx=7, n_rows=5), BADENUM, BADSIZE, BADENUM),
    ("evaluate", dict(ldx=0, D=0, n_rows=3), BADENUM, BADSIZE, BADENUM),
]

UNREGISTERED = [-1, 4, 5, USER_BASE - 1, USER_BASE + USER_CAPACITY - 1, USER_BASE + USER_CAPACITY, 1 << 20]


def test_argument_checks_return_before_any_device_work(lib, registered):
    objectives = [(0, 2)] + [(o, 3) for o in (1, 2, 3, registered)] + [(o, 4) for o in UNREGISTERED]
    launches = lib.evok_launch_count()
    failures = []
    for entry, change, *expected in CASES:
        args = {**BASE[entry], **change}
        for objective, col in objectives:
            want = expected[col - 2]
            got = call(lib, entry, objective, args)
            if got != want:
                failures.append(f"{entry}({objective}, {change}): {got}, expected {want}")
    assert not failures, "\n".join(failures)
    assert lib.evok_launch_count() == launches


# ------------------------------------------------------------------------------------------------ the kernel each call launches
KERNEL = re.compile(r"evok::(sample_eval_kernel|eval_kernel)<([^,<>]+(?:<\d+>)?), ([^>]*)>")


def launched_kernel(run, tmp_path):
    """(kernel name, accumulator, flag template arguments, block, grid) of the one kernel `run` launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    for _ in range(3):  # now and then the profiler delivers no kernel record from a window this short: take another
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                run()
            torch.cuda.synchronize()
        path = tmp_path / "trace.json"
        prof.export_chrome_trace(str(path))
        events = [e for e in json.loads(path.read_text())["traceEvents"] if e.get("cat") == "kernel"]
        if events:
            break
    launches = {(e["name"], tuple(e["args"]["block"]), tuple(e["args"]["grid"])) for e in events}
    assert len(launches) == 1 and len(events) <= 3, launches
    m = KERNEL.search(events[0]["name"])
    assert m, events[0]["name"]
    flags = tuple(v.strip() == "true" for v in m.group(3).split(","))
    return m.group(1), m.group(2), flags, tuple(events[0]["args"]["block"]), tuple(events[0]["args"]["grid"])


_fused = {}


def fused_objective():
    from evotorch_b200.objectives import FusedObjective

    if "o" not in _fused:
        _fused["o"] = FusedObjective("dispatch_quartic", {"s": "x**4 - x"}, "s")
    return _fused["o"]


OBJECTIVES = ["none", "sphere", "fused"]
LAYOUTS = ["vec", "odd_D", "mu_offset"]  # D = 64 aligned; D = 63; D = 64 with mu 4 bytes into its allocation


def operands(layout, n):
    import torch

    D = 63 if layout == "odd_D" else 64
    g = torch.Generator().manual_seed(D)
    mu_buf = (torch.rand(D + 1, generator=g) * 2 - 1).cuda()
    mu = mu_buf[1:] if layout == "mu_offset" else mu_buf[:D].clone()
    sigma = (torch.rand(D, generator=g) + 0.5).cuda()
    return D, mu, sigma, torch.empty(n, D, device="cuda"), torch.empty(n, device="cuda")


def objective_id(name):
    from evotorch_b200 import ops

    return fused_objective().evok_objective_id if name == "fused" else {"none": ops.OBJ_NONE, "sphere": ops.OBJ_SPHERE}[name]


def accumulator(name):
    return {"none": "evok::ObjAcc<0>", "sphere": "evok::ObjAcc<1>", "fused": "evok_user::Acc"}[name]


def sample_case(entry, name, layout, sym, store, n=2048):
    """A function that makes one sampler call, and the kernel it must launch: (name, accumulator, sym / store / vec / push / sq)."""
    import torch

    from evotorch_b200 import ops

    D, mu, sigma, X, f = operands(layout, n)
    obj = objective_id(name)
    Xa = X if store else None
    fa = None if name == "none" else f
    vec = layout == "vec"  # X = torch.empty(n, 64): aligned rows
    if entry == "sample_eval":
        run = lambda: ops.sample_eval(obj, Xa, mu, sigma, n_rows=n, symmetric=sym, seed=1, stream_id=2, f=fa)  # noqa: E731
        flags = (sym, store, vec, False, False)
    elif entry == "sample_eval_sq":
        q = torch.empty(n, device="cuda")
        run = lambda: ops.sample_eval_sq(obj, Xa, mu, sigma, q, n_rows=n, seed=1, stream_id=2, f=fa)  # noqa: E731
        flags = (False, store, vec, False, True)
    else:
        f_all = torch.empty(n, device="cuda")
        flag_words = torch.zeros(1, dtype=torch.int64, device="cuda")
        epoch = torch.zeros(1, dtype=torch.int64, device="cuda")
        done = torch.zeros(1, dtype=torch.int32, device="cuda")
        pf, pg = peers(f_all.data_ptr()), peers(flag_words.data_ptr())
        ops._load_objective(obj, mu)

        def run():
            rc = nat.lib().evok_sample_eval_push(obj, nat.ptr(Xa), 0 if Xa is None else D, mu.data_ptr(), sigma.data_ptr(), 0, n, D,
                                                 int(sym), 1, 2, None, 1, 0, pf, pg, epoch.data_ptr(), done.data_ptr(),
                                                 nat.stream_of(mu))
            nat.check(rc, "evok_sample_eval_push")

        flags = (sym, store, vec, True, False)
    return run, ("sample_eval_kernel", accumulator(name), flags)


def sampler_cases():
    out = []
    for name in OBJECTIVES:
        for layout in LAYOUTS:
            for store in (True, False):
                if name == "none" and not store:
                    continue  # nothing to sample into
                for sym in (False, True):
                    out.append(("sample_eval", name, layout, sym, store))
                    if name != "none":
                        out.append(("sample_eval_push", name, layout, sym, store))
                out.append(("sample_eval_sq", name, layout, False, store))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("entry,name,layout,sym,store", sampler_cases())
def test_sampler_launches_the_chosen_kernel(entry, name, layout, sym, store, tmp_path):
    run, want = sample_case(entry, name, layout, sym, store)
    run()  # loads a registered objective's module and warms up outside the profiled window
    kind, acc, flags, block, grid = launched_kernel(run, tmp_path)
    assert (kind, acc, flags) == want
    assert block == (256, 1, 1) and grid[1:] == (1, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["vec", "odd_D", "row_offset"])
@pytest.mark.parametrize("name", ["sphere", "fused"])
def test_evaluate_launches_the_chosen_kernel(name, layout, tmp_path):
    import torch

    from evotorch_b200 import ops

    n = 2048
    buf = torch.rand(n, 65, device="cuda")
    X = {"vec": buf[:, :64].contiguous(), "odd_D": buf[:, :63].contiguous(), "row_offset": buf[:, 1:]}[layout]
    obj = objective_id(name)
    ops.evaluate(obj, X)
    kind, acc, flags, block, grid = launched_kernel(lambda: ops.evaluate(obj, X), tmp_path)
    assert (kind, acc, flags) == ("eval_kernel", accumulator(name), (layout == "vec",))
    assert block == (256, 1, 1) and grid[1:] == (1, 1)
