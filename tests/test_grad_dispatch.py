"""How the gradient pass (K4) checks its arguments and which kernels it launches.

The CPU part maps argument combinations of evok_grad, _regen, _hybrid, _push and evok_sepcma_moments to return codes; every case
returns before a device is touched, so the launch count does not move (evok_grad_batched's codes sit with
evok_grad_batched_regen's in test_functional_fused_abi.py).  The GPU part runs each entry point under torch.profiler in a child
process and pins every kernel it launches, in order: name with template arguments, block and grid.  The plan is restated here, as
the bit-comparison tests give the same numbers for many plans and would not notice a wrong one."""

import ctypes
import json
import os
import subprocess
import sys

import pytest

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build

NULLPTR, BADSIZE, BADENUM, WORKSPACE, ODDROWS = -1, -2, -3, -4, -5  # EVOK_E_* of include/evok.h
MAX_PEERS = 16
P = 64  # any non-null pointer: the argument checks never dereference it
SYM, SEP, EXP, MOM = 1, 0, 2, 3  # EVOK_GRAD_*


@pytest.fixture(scope="module")
def lib():
    evok_build.build()
    return nat.lib()


def peers(ptrs):
    return None if ptrs is None else (ctypes.c_void_p * len(ptrs))(*ptrs)


# ws_bytes = 0: arguments that pass every check end at EVOK_E_WORKSPACE, before the empty case and any device work
BASE = dict(form=SYM, X=P, ldx=8, w=P, mu=P, sigma=P, row0=0, n_rows=4, D=8, out_mu=P, out_sigma=P, ws=P, split=0, world=2, rank=1,
            slots=(P, P), flags=(P, P), epoch=P, done=P)


def call(lib, entry, a):
    if entry == "grad":
        return lib.evok_grad(a["form"], a["X"], a["ldx"], a["w"], a["mu"], a["sigma"], a["n_rows"], a["D"], 1.0, 1.0, a["out_mu"], a["out_sigma"],
                             a["ws"], 0, None)
    if entry == "regen":
        return lib.evok_grad_regen(a["form"], a["w"], a["mu"], a["sigma"], a["row0"], a["n_rows"], a["D"], 0, 0, None, 1.0, 1.0, a["out_mu"],
                                   a["out_sigma"], a["ws"], 0, None)
    if entry == "hybrid":
        return lib.evok_grad_hybrid(a["form"], a["X"], a["ldx"], a["w"], a["mu"], a["sigma"], a["row0"], a["n_rows"], a["D"], 0, 0, None,
                                    a["split"], 1.0, 1.0, a["out_mu"], a["out_sigma"], a["ws"], 0, None)
    return lib.evok_grad_push(a["form"], a["X"], a["ldx"], a["w"], a["mu"], a["sigma"], a["row0"], a["n_rows"], a["D"], 0, 0, None, 1.0, 1.0,
                              a["world"], a["rank"], peers(a["slots"]), peers(a["flags"]), a["epoch"], a["done"], a["ws"], 0, None)


ENTRIES = ["grad", "regen", "hybrid", "push"]
# (changed arguments, code for evok_grad, _regen, _hybrid, _push)
CASES = [
    ({}, WORKSPACE, WORKSPACE, WORKSPACE, WORKSPACE),
    (dict(w=None), NULLPTR, NULLPTR, NULLPTR, NULLPTR),
    (dict(w=None, n_rows=0), WORKSPACE, WORKSPACE, WORKSPACE, WORKSPACE),  # an empty shard has no weights to point at
    (dict(mu=None), NULLPTR, NULLPTR, NULLPTR, NULLPTR),
    (dict(sigma=None), NULLPTR, NULLPTR, NULLPTR, NULLPTR),
    (dict(ws=None), NULLPTR, NULLPTR, NULLPTR, NULLPTR),
    (dict(out_mu=None), NULLPTR, NULLPTR, NULLPTR, WORKSPACE),  # the push writes into the peers' slots
    (dict(out_sigma=None), NULLPTR, NULLPTR, NULLPTR, WORKSPACE),
    (dict(X=None), NULLPTR, WORKSPACE, NULLPTR, WORKSPACE),  # the push regenerates the rows
    (dict(X=None, ldx=7), NULLPTR, WORKSPACE, NULLPTR, WORKSPACE),
    (dict(form=4), BADENUM, BADENUM, BADENUM, BADENUM),
    (dict(form=-1, n_rows=-2), BADENUM, BADENUM, BADENUM, BADENUM),
    (dict(n_rows=-2), BADSIZE, BADSIZE, BADSIZE, BADSIZE),
    (dict(D=0), BADSIZE, BADSIZE, BADSIZE, BADSIZE),
    (dict(row0=-2), WORKSPACE, BADSIZE, BADSIZE, BADSIZE),  # evok_grad has no first row
    (dict(ldx=7), BADSIZE, WORKSPACE, BADSIZE, BADSIZE),
    (dict(split=-2), WORKSPACE, WORKSPACE, BADSIZE, WORKSPACE),
    (dict(split=17), WORKSPACE, WORKSPACE, BADSIZE, WORKSPACE),
    (dict(split=16), WORKSPACE, WORKSPACE, WORKSPACE, WORKSPACE),
    (dict(split=-1), WORKSPACE, WORKSPACE, WORKSPACE, WORKSPACE),
    (dict(n_rows=3), ODDROWS, ODDROWS, ODDROWS, ODDROWS),
    (dict(row0=1), WORKSPACE, ODDROWS, ODDROWS, ODDROWS),
    (dict(n_rows=3, form=SEP), WORKSPACE, WORKSPACE, WORKSPACE, WORKSPACE),
    (dict(n_rows=3, ldx=7), BADSIZE, ODDROWS, BADSIZE, BADSIZE),
    (dict(slots=None), WORKSPACE, WORKSPACE, WORKSPACE, NULLPTR),
    (dict(flags=None), WORKSPACE, WORKSPACE, WORKSPACE, NULLPTR),
    (dict(epoch=None), WORKSPACE, WORKSPACE, WORKSPACE, NULLPTR),
    (dict(done=None), WORKSPACE, WORKSPACE, WORKSPACE, NULLPTR),
    (dict(slots=(P, None)), WORKSPACE, WORKSPACE, WORKSPACE, NULLPTR),
    (dict(flags=(None, P)), WORKSPACE, WORKSPACE, WORKSPACE, NULLPTR),
    (dict(world=0), WORKSPACE, WORKSPACE, WORKSPACE, BADSIZE),
    (dict(world=MAX_PEERS + 1), WORKSPACE, WORKSPACE, WORKSPACE, BADSIZE),
    (dict(rank=2), WORKSPACE, WORKSPACE, WORKSPACE, BADSIZE),
    (dict(rank=-1), WORKSPACE, WORKSPACE, WORKSPACE, BADSIZE),
    (dict(world=1, rank=0, slots=(P,), flags=(P,)), WORKSPACE, WORKSPACE, WORKSPACE, WORKSPACE),
    (dict(world=0, mu=None), NULLPTR, NULLPTR, NULLPTR, BADSIZE),  # the push checks its peers first
    (dict(slots=(P, None), n_rows=3), ODDROWS, ODDROWS, ODDROWS, NULLPTR),
]


def test_single_search_codes(lib):
    launches = lib.evok_launch_count()
    failures = []
    for change, *codes in CASES:
        for entry, want in zip(ENTRIES, codes):
            got = call(lib, entry, {**BASE, **change})
            if got != want:
                failures.append(f"{entry}({change}): {got}, expected {want}")
    assert not failures, "\n".join(failures)
    assert lib.evok_launch_count() == launches


SEPCMA_BASE = dict(aw=P, q=P, active=1, row0=0, n_rows=4, D=8, local=P, S2=P, wsum=P, ws=P)
SEPCMA_CASES = [
    ({}, WORKSPACE),
    (dict(aw=None), NULLPTR),
    (dict(q=None), NULLPTR),
    (dict(q=None, active=0), WORKSPACE),
    (dict(local=None), NULLPTR),
    (dict(S2=None), NULLPTR),
    (dict(wsum=None), NULLPTR),
    (dict(ws=None, n_rows=0), NULLPTR),
    (dict(n_rows=0), BADSIZE),  # no empty case here
    (dict(n_rows=-1), BADSIZE),
    (dict(D=0), BADSIZE),
    (dict(row0=-1), BADSIZE),
    (dict(row0=1, n_rows=3), WORKSPACE),
]


@pytest.mark.parametrize("changes,code", SEPCMA_CASES)
def test_sepcma_moments_codes(lib, changes, code):
    a = {**SEPCMA_BASE, **changes}
    before = lib.evok_launch_count()
    assert lib.evok_sepcma_moments(a["aw"], a["q"], a["active"], a["row0"], a["n_rows"], a["D"], 0, 0, None, a["local"], a["S2"], a["wsum"], a["ws"],
                                   0, None) == code
    assert lib.evok_launch_count() == before


# ------------------------------------------------------------------------------------------------ the kernels each call launches
SMS, CTAS_PER_SM, TMA_CTAS_PER_SM, UNROLL, MAX_GRID_Y = 132, 4, 3, 4, 65535


def _chunks(n_units, chunks):
    chunks = min(max(chunks, 1), 65535)
    upc = -(-n_units // chunks)
    return -(-n_units // upc)


def ldg_plan(n_units, D, vec, items=1, rebuild=False):
    """(tx, column tiles, row chunks) of the LDG kernel: plan_grad of csrc/evok_grad.cu restated."""
    col_threads = -(-D // vec)
    tx = 32
    while tx < 256 and tx < col_threads:
        tx *= 2
    tiles = -(-col_threads // tx)
    ty = 256 // tx
    n_chunks = _chunks(n_units, min(SMS * CTAS_PER_SM // tiles, -(-n_units // (ty * UNROLL * 16))))
    per_item = -(-SMS * CTAS_PER_SM // (tiles * items))
    if per_item < n_chunks:
        n_chunks = _chunks(n_units, per_item)
    if rebuild and vec == 1:
        tiles = -(-(-(-D // 4)) // tx)
    return tx, tiles, n_chunks


def tma_plan(n_units, D):
    tiles = -(-D // 1024)
    return tiles, _chunks(n_units, SMS * TMA_CTAS_PER_SM // tiles)


def b(v):
    return "true" if v else "false"


def ldg(vec, tx, sym, eps, tiles, chunks, items=1, sepw=False):
    return (f"grad_partial_kernel<{vec}, {tx}, {b(sym)}, {eps}, {b(sepw)}>", (256, 1, 1), (tiles, chunks, items))


def tma(sym, tiles, chunks):
    return (f"grad_partial_tma_kernel<{b(sym)}>", (288, 1, 1), (tiles, chunks, 1))


def fin(D, items=1, wsum=False):
    return (f"grad_finalize_kernel<{b(wsum)}>", (256, 1, 1), (-(-D // 256), items, 1))


def fin_push(D):
    return ("grad_finalize_push_kernel", (256, 1, 1), (-(-D // 256), 1, 1))


def single(form, n_rows, D, vec, eps=0):
    sym = form == SYM
    tx, tiles, chunks = ldg_plan(n_rows // 2 if sym else n_rows, D, vec)
    return [ldg(vec, tx, sym, eps, tiles, chunks), fin(D)]


def batched(form, items, n_rows, D, vec, eps=0):
    sym = form == SYM
    tx, tiles, chunks = ldg_plan(n_rows // 2 if sym else n_rows, D, vec, items, rebuild=eps == 2)
    out = []
    for b0 in range(0, items, MAX_GRID_Y):
        nb = min(MAX_GRID_Y, items - b0)
        out += [ldg(4 if eps else vec, tx, sym, eps, tiles, chunks, nb), fin(D, nb)]
    return out


def case_list():
    """(case id, expected launches); `make_case` builds the call of each id."""
    n, D = 8192, 1024
    push_tx, push_tiles, push_chunks = ldg_plan(500, 64, 4)  # 1000 symmetric rows
    cases = [
        ("tma_sym", [tma(True, *tma_plan(n // 2, D)), fin(D)]),
        ("tma_sep", [tma(False, *tma_plan(n, D)), fin(D)]),
        ("ldg_sym_tma_off", single(SYM, n, D, 4)),
        ("ldg_sep_tma_off", single(SEP, n, D, 4)),
        ("moments", single(MOM, n, D, 4)),
        ("odd_D", single(SYM, n, D - 1, 1)),
        ("x_offset", single(SEP, n, D, 1)),
        ("few_units", single(SYM, 8000, D, 4)),
        ("regen_sym", single(SYM, n, D, 4, eps=1)),
        ("regen_sep", single(EXP, n, 37, 4, eps=1)),
        ("hybrid_0", [tma(True, *tma_plan(n // 2, D)), fin(D)]),
        ("hybrid_5", [tma(True, *tma_plan(n // 2, D)), fin(D)]),
        ("hybrid_auto", [tma(True, *tma_plan(n // 2, D)), fin(D)]),
        ("push_read", [ldg(4, push_tx, True, 0, push_tiles, push_chunks), fin_push(64)]),
        ("push_regen", [ldg(4, push_tx, True, 1, push_tiles, push_chunks), fin_push(64)]),
        ("push_empty", [fin_push(64)]),
        ("empty", []),
        ("empty_batched", []),
    ]
    tx, tiles, chunks = ldg_plan(1000, 8, 4)
    cases += [(f"sepcma_{act}", [ldg(4, tx, False, 1, tiles, chunks, sepw=True), fin(8, wsum=True)]) for act in ("active", "plain")]
    for d in (36, 37):
        vec = 4 if d % 4 == 0 else 1
        for items in (1, 3):
            for shared in (True, False):
                cases.append((f"batched_{d}_{items}_{'shared' if shared else 'items'}", batched(SEP, items, 1000, d, vec)))
        cases.append((f"batched_regen_{d}", batched(SYM, 3, 1000, d, vec, eps=2)))
    # one item at the TMA shape of a single search: a batch keeps the LDG plan (and so the rebuild's bits)
    cases += [("batched_wide_sym", batched(SYM, 1, n, D, 4)), ("batched_wide_sep", batched(SEP, 1, n, D, 4))]
    cases.append(("two_item_chunks", batched(SEP, 65536, 4, 4, 4)))
    return cases


def make_case(case_id):
    """A function that makes the call of `case_id` (operands made here, outside the profiled window), and EVOK_GRAD_TMA for it."""
    import torch

    from evotorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *s: torch.rand(*s, device="cuda", generator=g)  # noqa: E731
    env = "0" if case_id.endswith("tma_off") else None
    n, D = 8192, 1024
    form = {"sep": SEP, "moments": MOM, "x_offset": SEP}.get(case_id.split("_")[1] if case_id.startswith("ldg") else case_id, SYM)
    if case_id.startswith(("tma", "ldg", "moments", "odd_D", "x_offset", "few_units")):
        if case_id.startswith("tma"):
            form = SYM if case_id == "tma_sym" else SEP
        n = 8000 if case_id == "few_units" else n
        d = D - 1 if case_id == "odd_D" else D
        X = (rnd(n * d + 1)[1:] if case_id == "x_offset" else rnd(n * d)).view(n, d)
        w, mu, sigma = rnd(n) - 0.5, rnd(d), rnd(d) + 0.5
        return (lambda: ops.grad(form, X, w, mu, sigma, 1.0, 1.0)), env
    if case_id.startswith("regen"):
        form, d = (SYM, D) if case_id == "regen_sym" else (EXP, 37)
        w, mu, sigma = rnd(n) - 0.5, rnd(d), rnd(d) + 0.5
        return (lambda: ops.grad_regen(form, w, mu, sigma, seed=3, stream_id=4, row0=0, scale_mu=1.0, scale_sigma=1.0)), env
    if case_id.startswith("hybrid"):
        split = {"hybrid_0": 0, "hybrid_5": 5, "hybrid_auto": -1}[case_id]
        X, w, mu, sigma = rnd(n, D), rnd(n) - 0.5, rnd(D), rnd(D) + 0.5
        return (lambda: ops.grad_hybrid(SYM, X, w, mu, sigma, seed=3, stream_id=4, row0=0, scale_mu=1.0, scale_sigma=1.0, split=split)), env
    if case_id.startswith("push"):
        rows, d = (0 if case_id == "push_empty" else 1000), 64
        X = rnd(rows, d) if case_id == "push_read" else None
        w, mu, sigma = rnd(rows) - 0.5, rnd(d), rnd(d) + 0.5
        slots, flags = torch.empty(2 * d, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
        epoch, done = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
        ws = torch.empty(nat.lib().evok_grad_workspace_bytes(rows, d), dtype=torch.uint8, device="cuda")
        sp, fp = peers([slots.data_ptr()]), peers([flags.data_ptr()])

        def run():
            nat.check(nat.lib().evok_grad_push(SYM, nat.ptr(X), d, nat.ptr(w), mu.data_ptr(), sigma.data_ptr(), 0, rows, d, 3, 4, None, 1.0, 1.0, 1, 0,
                                               sp, fp, epoch.data_ptr(), done.data_ptr(), ws.data_ptr(), ws.numel(), nat.stream_of(mu)),
                      "evok_grad_push")

        return run, env
    if case_id.startswith("empty"):
        # zero rows through the C ABI: a tensor without elements has no data pointer, and X must not be NULL here
        mu, sigma, out = rnd(64), rnd(64), rnd(2, 3, 64)
        ws = torch.empty(nat.lib().evok_grad_batched_workspace_bytes(3, 0, 64), dtype=torch.uint8, device="cuda")
        X, w = mu.data_ptr(), sigma.data_ptr()

        def run():
            if case_id == "empty":
                rc = nat.lib().evok_grad(SYM, X, 64, w, mu.data_ptr(), sigma.data_ptr(), 0, 64, 1.0, 1.0, out[0].data_ptr(), out[1].data_ptr(),
                                         ws.data_ptr(), ws.numel(), nat.stream_of(mu))
            else:
                rc = nat.lib().evok_grad_batched(SYM, X, 0, 64, w, mu.data_ptr(), 0, sigma.data_ptr(), 0, 3, 0, 64, 1.0, 1.0, out[0].data_ptr(),
                                                 out[1].data_ptr(), ws.data_ptr(), ws.numel(), nat.stream_of(mu))
            nat.check(rc, case_id)
            assert not out[:, : 1 if case_id == "empty" else 3].any()  # the outputs are zeroed

        return run, env
    if case_id.startswith("sepcma"):
        aw, q = rnd(1000) - 0.5, rnd(1000) + 1.0
        active = case_id == "sepcma_active"
        return (lambda: ops.sepcma_moments(aw, q, active, 8, seed=3, stream_id=4)), env
    if case_id.startswith("batched_wide"):
        form = SYM if case_id == "batched_wide_sym" else SEP
        X, w = rnd(1, n, D), rnd(1, n) - 0.5
        mu, sigma = (rnd(D), rnd(D) + 0.5) if form == SYM else (rnd(1, D), rnd(1, D) + 0.5)
        return (lambda: ops.grad_batched(form, X, w, mu, sigma, 1.0, 1.0)), env
    if case_id.startswith("batched_regen"):
        d = int(case_id.split("_")[-1])
        w, mu, sigma = rnd(3, 1000) - 0.5, rnd(3, d), rnd(d) + 0.5
        return (lambda: ops.grad_batched_regen(SYM, w, mu, sigma, 1.0, 1.0, seed=3, stream_id0=4)), env
    if case_id.startswith("batched"):
        _, d, items, kind = case_id.split("_")
        d, items = int(d), int(items)
        X, w = rnd(items, 1000, d), rnd(items, 1000) - 0.5
        mu, sigma = (rnd(d), rnd(d) + 0.5) if kind == "shared" else (rnd(items, d), rnd(items, d) + 0.5)
        return (lambda: ops.grad_batched(SEP, X, w, mu, sigma, 1.0, 1.0)), env
    assert case_id == "two_item_chunks", case_id
    X, w, mu, sigma = rnd(65536, 4, 4), rnd(65536, 4) - 0.5, rnd(4), rnd(4) + 0.5
    return (lambda: ops.grad_batched(SEP, X, w, mu, sigma, 1.0, 1.0)), env


def profile_cases(path):
    """Child process: every case once to warm up and once counted, then all of them in one profiler window, kernels in order."""
    import re

    import torch
    from torch.profiler import ProfilerActivity, profile

    runs, out = [], {}
    for cid, _ in case_list():
        run, env = make_case(cid)
        runs.append((cid, run, env))

    def with_env(env, fn):  # the child starts without EVOK_GRAD_TMA
        if env is not None:
            os.environ["EVOK_GRAD_TMA"] = env
        fn()
        os.environ.pop("EVOK_GRAD_TMA", None)

    for cid, run, env in runs:
        with_env(env, run)
        before = nat.lib().evok_launch_count()
        with_env(env, run)
        out[cid] = {"count": nat.lib().evok_launch_count() - before}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for cid, run, env in runs:
            with_env(env, run)
        torch.cuda.synchronize()
    prof.export_chrome_trace(path + ".trace.json")
    with open(path + ".trace.json") as fh:
        events = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel" and "evok::" in e["name"]]
    events.sort(key=lambda e: e["ts"])
    pat = re.compile(r"evok::(\w+(?:<[^()]*>)?)\(")
    i = 0
    for cid, _, _ in runs:
        k = out[cid]["count"]
        out[cid]["kernels"] = [[pat.search(e["name"]).group(1), e["args"]["block"], e["args"]["grid"]] for e in events[i:i + k]]
        i += k
    out["_total"] = len(events)
    with open(path, "w") as fh:
        json.dump(out, fh)


@pytest.fixture(scope="module")
def launched(tmp_path_factory):
    """{case id: {"count": evok_launch_count delta, "kernels": [[name, block, grid], ...]}} from a child process.  The profiler runs
    there, never in the test process: a CUPTI session that ends in a process can leave later profiler windows without records."""
    here = os.path.dirname(os.path.abspath(__file__))
    path = str(tmp_path_factory.mktemp("grad_dispatch") / "launched.json")
    code = f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; import test_grad_dispatch as t; t.profile_cases({path!r})"
    env = {k: v for k, v in os.environ.items() if k != "EVOK_GRAD_TMA"}
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    with open(path) as fh:
        return json.load(fh)


@pytest.mark.gpu
@pytest.mark.parametrize("case_id,want", case_list(), ids=[c[0] for c in case_list()])
def test_launches(launched, case_id, want):
    got = launched[case_id]
    assert got["count"] == len(want), got
    assert [(k, tuple(bl), tuple(gr)) for k, bl, gr in got["kernels"]] == want


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 37])
@pytest.mark.parametrize("form", [SEP, SYM, EXP, MOM])
def test_one_item_batch_is_a_single_search(form, D):
    """The batched path with one item runs the single search's kernel with its plan, so it gives the same bits."""
    import torch

    from evotorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(D + form)
    n = 3000
    X = torch.randn(n, D, device="cuda", generator=g)
    w = torch.randn(n, device="cuda", generator=g)
    mu, sigma = torch.randn(D, device="cuda", generator=g), torch.rand(D, device="cuda", generator=g) + 0.5
    one = ops.grad(form, X, w, mu, sigma, 0.5, 0.25)
    batch = ops.grad_batched(form, X[None], w[None], mu, sigma, 0.5, 0.25)
    assert torch.equal(batch[0][0], one[0]) and torch.equal(batch[1][0], one[1])


@pytest.mark.gpu
def test_grad_batched_rejects_bad_operands():
    import torch

    from evotorch_b200 import ops

    B, n, d = 3, 16, 8
    X, w, mu, sigma = torch.rand(B, n, d, device="cuda"), torch.rand(B, n, device="cuda"), torch.rand(d, device="cuda"), torch.rand(d, device="cuda")
    for bad_w in (w.double(), w.cpu(), torch.rand(n, B, device="cuda").t()):
        with pytest.raises(ValueError, match="w"):
            ops.grad_batched(SEP, X, bad_w, mu, sigma, 1.0, 1.0)
    with pytest.raises(ValueError, match="number of items"):
        ops.grad_batched(SEP, X, w, torch.rand(2, d, device="cuda"), sigma, 1.0, 1.0)
    with pytest.raises(ValueError, match="number of items"):
        ops.grad_batched(SEP, X, w, mu, torch.rand(2, d, device="cuda"), 1.0, 1.0)
    ops.grad_batched(SEP, X, w, mu, sigma, 1.0, 1.0)  # and the well-formed call runs
