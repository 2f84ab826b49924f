"""The peer exchange at world sizes 2-16, simulated on one GPU.

Every rank of the exchange is a `PeerExchange` laid out over a plain device buffer of this GPU, with its own stream, epochs and
counters: the kernels take raw device pointers, so R buffers on one device are R "peers" to them, and the production entry points
(`ops.sample_eval_push`, `ops.grad_push`, `PeerExchange.push_fitness / wait_fitness / reduce_gradients / rank_sharded`) run
unchanged.  Each result is compared with the unsharded kernels (bit for bit) and with a float64 restatement.

Every buffer sits between guard regions, and its padding between sections, filled with a NaN sentinel that no kernel writes.

Concurrency: only the consumers spin (flag wait, slot reduction, the merge of the sharded ranking).  The host enqueues all producers
of an exchange point before any consumer of it, so no consumer sits ahead of a producer it waits for in a hardware queue, and
the spinning CTAs stay far below a full GPU (at most 16 x 8 CTAs of 256 threads).  Every wait has a 10 s time-out that raises the
error flag, which the tests check: a lost flag fails, it does not hang.  What one GPU cannot cover: ordering over NVLink between
GPUs, and CUDA-graph capture of a multi-rank generation.
"""

import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from evotorch_b200 import _native as nat
    from evotorch_b200 import ops
    from evotorch_b200.distributed import shard_rows
    from evotorch_b200.distributions import ExpSeparableGaussian, SeparableGaussian, SymmetricSeparableGaussian
    from evotorch_b200.peer import PeerExchange

DEV = "cuda"
TIMEOUT_NS = 10_000_000_000
GUARD = 4096  # bytes of sentinel before and after every exchange buffer
SENTINEL = 0x7FC0DEAD  # a quiet NaN that no kernel produces
POPSIZE = 20_000
# an empty shard, one-row shards and odd first rows; the symmetric one keeps every count and first row even
UNEVEN = [7, 0, 12001, 30, 1, 600, 2, 2050]
UNEVEN_SYM = [6, 0, 12002, 30, 2, 600, 2, 2050]
LAYOUTS = ["2", "3", "8", "16", "uneven"]
OBJECTIVES = ["sphere", "rastrigin", "ackley"]
DIMS = {"sphere": 64, "rastrigin": 37, "ackley": 100}  # vectorised and scalar sampler paths
FORMS = ["symmetric", "separable", "exp", "moments"]
E_NULLPTR, E_BADSIZE = -1, -2  # EVOK_E_* of include/evok.h


def counts_of(layout: str, symmetric: bool) -> list:
    if layout == "uneven":
        return list(UNEVEN_SYM if symmetric else UNEVEN)
    return shard_rows(POPSIZE, int(layout), 0, symmetric)[2]


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


class SimWorld:
    """R ranks of one peer exchange on this GPU, shard r = rows [row0[r], row0[r] + counts[r])."""

    def __init__(self, counts: list, D: int):
        self.counts, self.D = list(counts), int(D)
        self.R, self.N = len(counts), sum(counts)
        self.row0 = [sum(counts[:r]) for r in range(self.R)]
        self.streams = [torch.cuda.Stream() for _ in range(self.R)]
        self.px, self.raw = [], []
        for r in range(self.R):
            px = PeerExchange.__new__(PeerExchange)
            px._configure(self.N, self.D, DEV, r, self.R, TIMEOUT_NS)
            self.px.append(px)
            self.raw.append(torch.full(((2 * GUARD + px.nbytes) // 4,), SENTINEL, dtype=torch.int32, device=DEV))
        bases = [b.data_ptr() + GUARD for b in self.raw]
        p0 = self.px[0]
        # the sections the protocol writes, in 4-byte words of the raw buffer; everything else must keep the sentinel
        sections = [(p0._off_f, 4 * self.N), (p0._off_slots, 8 * self.R * self.D), (p0._off_flags_f, 8 * self.R),
                    (p0._off_flags_g, 8 * self.R), (p0._off_keys, 4 * self.N), (p0._off_fsum, 8 * self.R)]
        self.outside = torch.ones_like(self.raw[0], dtype=torch.bool)
        for off, nbytes in sections:
            self.outside[(GUARD + off) // 4:(GUARD + off + nbytes) // 4] = False
        for r, px in enumerate(self.px):
            for off in (p0._off_flags_f, p0._off_flags_g):
                self.raw[r][(GUARD + off) // 4:(GUARD + off + 8 * self.R) // 4].zero_()  # as evok_peer_alloc leaves them
            px._lay_out(bases[r], bases)
        torch.cuda.synchronize()

    def on(self, r: int):
        return torch.cuda.stream(self.streams[r])

    def producers_done(self) -> None:
        """Order every rank's next work after every rank's work so far (an event per stream, waited on by every stream)."""
        events = []
        for s in self.streams:
            e = torch.cuda.Event()
            e.record(s)
            events.append(e)
        for s in self.streams:
            for e in events:
                s.wait_event(e)

    def poison(self) -> None:
        for px in self.px:
            bits(px.f_all).fill_(SENTINEL)
            bits(px.slots).fill_(SENTINEL)
        torch.cuda.synchronize()

    def flags(self, r: int, which: str) -> torch.Tensor:
        px = self.px[r]
        off = px._off_flags_f if which == "f" else px._off_flags_g
        return self.raw[r].view(torch.int64)[(GUARD + off) // 8:(GUARD + off) // 8 + self.R]

    def check(self, epoch_f: int, epoch_g: int, f_written: bool = True) -> None:
        """After a synchronisation: guards and padding untouched, every row of every f_all written, no time-out, every epoch and
        flag at the number of completed exchanges and every completion counter back at 0."""
        torch.cuda.synchronize()
        for r, px in enumerate(self.px):
            assert bool((self.raw[r][self.outside] == SENTINEL).all()), f"rank {r}: a write landed outside the exchange sections"
            if f_written:
                assert not bool(torch.isnan(px.f_all).any()), f"rank {r}: rows of f_all that no shard wrote"
            assert px._counters.tolist() == [0, 0, 0, 0], (r, px._counters.tolist())
            assert px._rank_counters.tolist() == [0, 0, 0, 0], (r, px._rank_counters.tolist())
            assert px._epochs.tolist() == [epoch_f, epoch_g], (r, px._epochs.tolist())
            assert self.flags(r, "f").tolist() == [epoch_f] * self.R, (r, self.flags(r, "f").tolist())
            assert self.flags(r, "g").tolist() == [epoch_g] * self.R, (r, self.flags(r, "g").tolist())


def f64_objective(objective: str, X: torch.Tensor) -> torch.Tensor:
    X = X.double()
    D = X.shape[1]
    if objective == "sphere":
        return (X**2).sum(1)
    if objective == "rastrigin":
        return 10.0 * D + (X**2 - 10 * torch.cos(2 * math.pi * X)).sum(1)
    return -20 * torch.exp(-0.2 * torch.sqrt((X**2).mean(1))) - torch.exp(torch.cos(2 * math.pi * X).mean(1)) + 20 + math.e


def distribution_params(D: int, seed: int) -> tuple:
    g = torch.Generator(device="cpu").manual_seed(seed)
    mu = (torch.rand(D, generator=g) * 4 - 2).to(DEV)
    sigma = (torch.rand(D, generator=g) + 0.5).to(DEV)
    return mu, sigma


# ------------------------------------------------------------------------------------------------ (a) / (b) fitness gather
def check_gathered(world: SimWorld, objective: str, symmetric: bool, X_shards: list, mu, sigma, seed: int, stream_id: int,
                   stream_offset) -> None:
    N, D = world.N, world.D
    oid = ops.OBJECTIVE_IDS[objective]
    X = torch.empty(N, D, device=DEV)
    f = torch.empty(N, device=DEV)
    ops.sample_eval(oid, X, mu, sigma, n_rows=N, symmetric=symmetric, seed=seed, stream_id=stream_id, f=f, stream_offset=stream_offset)
    torch.cuda.synchronize()
    for r, px in enumerate(world.px):
        assert same_bits(px.f_all, f), f"rank {r}: gathered fitnesses differ from the unsharded sampler"
        if X_shards[r] is not None:
            assert same_bits(X_shards[r], X[world.row0[r]:world.row0[r] + world.counts[r]]), f"rank {r}: shard != rows of the population"
    # the tolerance of test_fused_sample_eval_is_consistent
    torch.testing.assert_close(f.double(), f64_objective(objective, X), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("stream_offset", [False, True])
@pytest.mark.parametrize("objective", OBJECTIVES)
@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_fitness_gather_pushed_from_the_sampler(layout, symmetric, lazy, objective, stream_offset):
    """Round-1 protocol: every shard's sampler stores its fitnesses into every rank's f_all, then every rank waits."""
    counts = counts_of(layout, symmetric)
    D = DIMS[objective]
    world = SimWorld(counts, D)
    mu, sigma = distribution_params(D, len(counts) + D)
    off = torch.tensor([3], dtype=torch.int32, device=DEV) if stream_offset else None
    seed, sid = 0x5EED_0000_1234 + D, 11
    world.poison()
    X_shards = []
    for r, px in enumerate(world.px):
        with world.on(r):
            Xr = None if lazy else torch.empty(counts[r], D, device=DEV)
            ops.sample_eval_push(ops.OBJECTIVE_IDS[objective], Xr, mu, sigma, n_rows=counts[r], symmetric=symmetric, seed=seed,
                                 stream_id=sid, row0=world.row0[r], peer=px, stream_offset=off)
        X_shards.append(Xr)
    world.producers_done()
    for r, px in enumerate(world.px):
        with world.on(r):
            px.wait_fitness()
    world.check(1, 0)
    check_gathered(world, objective, symmetric, X_shards, mu, sigma, seed, sid, off)


def push_paths(counts: list) -> set:
    """The copy loops of peer_push_kernel that a layout reaches: 16-byte vectors (+ a byte tail), or 4-byte words."""
    paths, row0 = set(), 0
    for n in counts:
        if n:
            paths.add(("vec+tail" if n % 4 else "vec") if row0 % 4 == 0 else "word")
        row0 += n
    return paths


@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_fitness_gather_by_the_push_kernel(layout, symmetric, lazy):
    """Round-2 protocol (the default): the plain sampler writes the rank's slice of its own f_all, `push_fitness` copies it to
    every peer and raises the flag."""
    counts = counts_of(layout, symmetric)
    if layout == "uneven" and not symmetric:
        assert push_paths(counts) >= {"vec+tail", "word"}
    objective = OBJECTIVES[LAYOUTS.index(layout) % 3]
    D = DIMS[objective]
    world = SimWorld(counts, D)
    mu, sigma = distribution_params(D, 2 * len(counts) + D)
    seed, sid = 0xC0FFEE + D, 5
    world.poison()
    X_shards = []
    for gen in range(2):  # twice: the second exchange runs on the counters the first one left
        for r, px in enumerate(world.px):
            lo, n = world.row0[r], counts[r]
            with world.on(r):
                Xr = None if lazy else torch.empty(n, D, device=DEV)
                ops.sample_eval(ops.OBJECTIVE_IDS[objective], Xr, mu, sigma, n_rows=n, symmetric=symmetric, seed=seed, stream_id=sid + gen,
                                row0=lo, f=px.f_all[lo:lo + n])
                px.push_fitness(lo, n)
            if gen == 1:
                X_shards.append(Xr)
        world.producers_done()
        for r, px in enumerate(world.px):
            with world.on(r):
                px.wait_fitness()
        world.check(gen + 1, 0)
        if gen == 0:
            world.poison()
    check_gathered(world, objective, symmetric, X_shards, mu, sigma, seed, sid + 1, None)


# ------------------------------------------------------------------------------------------------ (c) gradient all-reduce
def f64_gradient(form: str, X: torch.Tensor, w: torch.Tensor, mu, sigma, scale_mu: float, scale_sigma: float) -> tuple:
    """The float64 gradient of the whole population and the tolerances of test_grad_kernel_matches_oracle_ragged_shapes."""
    X64, w64, mu64, sg64 = X.double(), w.double(), mu.double(), sigma.double()
    if form == "symmetric":
        eps = X64[0::2] - mu64
        a, b = (w64[0::2] - w64[1::2]) / 2, (w64[0::2] + w64[1::2]) / 2
        g = (eps**2 - sg64**2) / sg64
    else:
        eps = X64 - mu64
        a = b = w64
        g = {"separable": (eps**2 - sg64**2) / sg64, "exp": (eps / sg64) ** 2 - 1, "moments": eps**2}[form]
    ref_m = scale_mu * (a[:, None] * eps).sum(0)
    ref_s = scale_sigma * (b[:, None] * g).sum(0)
    tol_m = 3e-6 * abs(scale_mu) * float((a.abs()[:, None] * eps.abs()).sum(0).max()) + 1e-9
    tol_s = 3e-6 * abs(scale_sigma) * float((b.abs()[:, None] * (g.abs() + 1)).sum(0).max()) + 1e-9
    return ref_m, ref_s, tol_m, tol_s


GRAD_CASES = [("2", 1024), ("3", 515), ("8", 1), ("16", 1024), ("uneven", 515), ("uneven", 1)]


@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("layout,D", GRAD_CASES)
def test_gradient_all_reduce(layout, D, form, lazy):
    """`grad_push` on every shard then `reduce_gradients`: bit-identical on every rank, bit-identical to the rank-order fp32 sum
    of the unsharded kernel on each shard, and close to the float64 gradient of the whole population.  At D = 1024 over two
    ranks the shards are >= 4096 units, so the TMA-staged gradient kernel runs inside the push."""
    symmetric = form == "symmetric"
    fid = getattr(ops, "GRAD_" + form.upper())
    counts = counts_of(layout, symmetric)
    world = SimWorld(counts, D)
    N = world.N
    mu, sigma = distribution_params(D, N + D + fid)
    seed, sid = 0xABCDEF + D, 3
    X = torch.empty(N, D, device=DEV)
    ops.sample_eval(ops.OBJ_NONE, X, mu, sigma, n_rows=N, symmetric=symmetric, seed=seed, stream_id=sid)
    g = torch.Generator(device=DEV).manual_seed(N + D)
    if form == "moments":
        w = (torch.rand(N, device=DEV, generator=g) < 0.3).float()  # a 0/1 elite mask, as CEM uses
    else:
        w = torch.randn(N, device=DEV, generator=g) / N
    smu, ssig = 0.5, 2.0
    shards = [X[lo:lo + n].clone() for lo, n in zip(world.row0, counts)]
    torch.cuda.synchronize()
    world.poison()
    for r, px in enumerate(world.px):
        lo, n = world.row0[r], counts[r]
        with world.on(r):
            ops.grad_push(fid, None if lazy else shards[r], w[lo:lo + n], mu, sigma, scale_mu=smu, scale_sigma=ssig, peer=px, seed=seed,
                          stream_id=sid, row0=lo)
    world.producers_done()
    for r, px in enumerate(world.px):
        with world.on(r):
            px.reduce_gradients()
    world.check(0, 1, f_written=False)
    # the unsharded kernel on each shard, summed in rank order in fp32
    parts = []
    for r in range(world.R):
        lo, n = world.row0[r], counts[r]
        if n == 0:  # an empty shard contributes zeros (its weights have no data pointer)
            pm, ps = ops.grad_regen(fid, torch.empty(0, device=DEV), mu, sigma, seed=seed, stream_id=sid, row0=lo, scale_mu=smu, scale_sigma=ssig)
            assert not bool(torch.cat([pm, ps]).any())
        elif lazy:
            pm, ps = ops.grad_regen(fid, w[lo:lo + n], mu, sigma, seed=seed, stream_id=sid, row0=lo, scale_mu=smu, scale_sigma=ssig)
        else:
            pm, ps = ops.grad(fid, shards[r], w[lo:lo + n], mu, sigma, smu, ssig)
        parts.append(torch.cat([pm, ps]))
    acc = torch.zeros(2 * D, device=DEV)
    for p in parts:
        acc = acc + p
    torch.cuda.synchronize()
    for r, px in enumerate(world.px):
        assert same_bits(px.slots, torch.cat(parts)), f"rank {r}: slot s must hold shard s's partial gradient"
        assert same_bits(px.reduced, world.px[0].reduced), f"rank {r} reduced to other bits than rank 0"
        assert same_bits(px.reduced, acc), f"rank {r}: not the rank-order sum of the shards' gradients"
    ref_m, ref_s, tol_m, tol_s = f64_gradient(form, X, w, mu, sigma, smu, ssig)
    torch.testing.assert_close(acc[:D].double(), ref_m, rtol=1e-4, atol=tol_m)
    torch.testing.assert_close(acc[D:].double(), ref_s, rtol=1e-4, atol=tol_s)


# ------------------------------------------------------------------------------------------------ (d) back-to-back generations
@pytest.mark.parametrize("push", ["sampler", "kernel"])
@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("layout", ["3", "uneven"])
def test_back_to_back_generations_without_host_synchronisation(layout, lazy, push):
    """Whole generations (push, wait, rank, grad_push, reduce, ClipUp on each rank's own mu) enqueued back to back with no host
    synchronisation and no events between the ranks.  The rank with the largest shard sleeps about a millisecond before each of
    its consumers, so the others run into the next generation and overwrite its f_all and slots as early as the protocol lets
    them: if a buffer were rewritten before its reader passed the other exchange point (DESIGN.md section 5: no double
    buffering), a generation's copy would differ from the single-rank run."""
    gens, D, objective = 4, 256, ops.OBJ_RASTRIGIN
    counts = counts_of(layout, True)
    world = SimWorld(counts, D)
    R, N = world.R, world.N
    slow = max(range(R), key=lambda r: counts[r])
    mu0, sigma = distribution_params(D, 7 * R)
    seed, scale = 0xFEED, 2.0 / N
    world.poison()
    mus = [mu0.clone() for _ in range(R)]
    vels = [torch.zeros(D, device=DEV) for _ in range(R)]
    out_f = [torch.empty(gens, N, device=DEV) for _ in range(R)]
    out_g = [torch.empty(gens, 2 * D, device=DEV) for _ in range(R)]
    Xs = [None if lazy else torch.empty(n, D, device=DEV) for n in counts]
    torch.cuda.synchronize()
    for gen in range(gens):
        for r, px in enumerate(world.px):
            lo, n = world.row0[r], counts[r]
            with world.on(r):
                if push == "sampler":
                    ops.sample_eval_push(objective, Xs[r], mus[r], sigma, n_rows=n, symmetric=True, seed=seed, stream_id=gen, row0=lo, peer=px)
                else:
                    ops.sample_eval(objective, Xs[r], mus[r], sigma, n_rows=n, symmetric=True, seed=seed, stream_id=gen, row0=lo,
                                    f=px.f_all[lo:lo + n])
                    px.push_fitness(lo, n)
        for r, px in enumerate(world.px):
            lo, n = world.row0[r], counts[r]
            with world.on(r):
                if r == slow:
                    torch.cuda._sleep(2_000_000)
                f_all = px.wait_fitness()
                out_f[r][gen].copy_(f_all)  # before this rank's gradient push: after it, the peers may overwrite f_all
                w = ops.rank(f_all, "centered", False)
                ops.grad_push(ops.GRAD_SYMMETRIC, Xs[r], w[lo:lo + n], mus[r], sigma, scale_mu=scale, scale_sigma=scale, peer=px, seed=seed,
                              stream_id=gen, row0=lo)
        for r, px in enumerate(world.px):
            with world.on(r):
                if r == slow:
                    torch.cuda._sleep(2_000_000)
                gm, _ = px.reduce_gradients()
                out_g[r][gen].copy_(px.reduced)
                ops.clipup_step(gm, vels[r], 0.3, 0.9, 0.5, mu=mus[r])
    world.check(gens, gens)
    # the same generations on one rank
    mu, vel = mu0.clone(), torch.zeros(D, device=DEV)
    X, f = torch.empty(N, D, device=DEV), torch.empty(N, device=DEV)
    for gen in range(gens):
        ops.sample_eval(objective, None if lazy else X, mu, sigma, n_rows=N, symmetric=True, seed=seed, stream_id=gen, f=f)
        w = ops.rank(f, "centered", False)
        acc = torch.zeros(2 * D, device=DEV)
        for lo, n in zip(world.row0, counts):
            if n == 0:
                continue
            if lazy:
                pm, ps = ops.grad_regen(ops.GRAD_SYMMETRIC, w[lo:lo + n], mu, sigma, seed=seed, stream_id=gen, row0=lo, scale_mu=scale,
                                        scale_sigma=scale)
            else:
                pm, ps = ops.grad(ops.GRAD_SYMMETRIC, X[lo:lo + n].clone(), w[lo:lo + n], mu, sigma, scale, scale)
            acc = acc + torch.cat([pm, ps])
        for r in range(R):
            assert same_bits(out_f[r][gen], f), f"generation {gen}, rank {r}: f_all"
            assert same_bits(out_g[r][gen], acc), f"generation {gen}, rank {r}: reduced gradient"
        ops.clipup_step(acc[:D].contiguous(), vel, 0.3, 0.9, 0.5, mu=mu)
    torch.cuda.synchronize()
    for r in range(R):
        assert same_bits(mus[r], mus[0]), f"rank {r}: mu diverged from rank 0"
    assert same_bits(mus[0], mu)


# ------------------------------------------------------------------------------------------------ (e) sharded ranking -> gradient
@pytest.mark.parametrize("method", ["centered", "linear", "nes"])
@pytest.mark.parametrize("dist_name", ["symmetric", "separable", "exp"])
@pytest.mark.parametrize("layout", ["2", "3", "uneven"])
def test_sharded_ranking_into_the_gradient(layout, dist_name, method):
    """`rank_sharded`'s local utilities into `partial_gradients(..., local_weights_of=N, peer=)` and `finalize_gradients` (the
    EVOTORCH_B200_SHARDED_RANK=1 path of the sharded generation): bit-identical to the replicated path on slices of the global
    ranking, and close to `compute_gradients` on the whole population.  The pairs `accepts_local_weights` refuses must raise."""
    cls = {"symmetric": SymmetricSeparableGaussian, "separable": SeparableGaussian, "exp": ExpSeparableGaussian}[dist_name]
    symmetric = dist_name == "symmetric"
    D = 129
    counts = counts_of(layout, symmetric)
    mu, sigma = distribution_params(D, len(counts) + 1)
    extra = {} if dist_name == "exp" else {"divide_mu_grad_by": "num_solutions", "divide_sigma_grad_by": "num_solutions"}
    dist = cls({"mu": mu, "sigma": sigma, **extra})
    if not dist.accepts_local_weights(method):
        with pytest.raises(ValueError, match="whole population"):
            dist.partial_gradients(torch.empty(4, D, device=DEV), torch.zeros(4, device=DEV), 0, method, local_weights_of=8)
        return
    world = SimWorld(counts, D)
    N = world.N
    X, f = torch.empty(N, D, device=DEV), torch.empty(N, device=DEV)
    ops.sample_eval(ops.OBJ_RASTRIGIN, X, mu, sigma, n_rows=N, symmetric=symmetric, seed=99, stream_id=4, f=f)
    f = torch.round(f * 4) / 4  # ties within and across shards
    offsets = world.row0 + [N]
    shards = [X[lo:lo + n].clone() for lo, n in zip(world.row0, counts)]
    for r, px in enumerate(world.px):
        lo, n = world.row0[r], counts[r]
        px.f_all[lo:lo + n].copy_(f[lo:lo + n])  # the shard's fitness column is its slice of the exchange buffer
    torch.cuda.synchronize()
    # Each call below ends its stream's work with a spinning consumer (the merge, the slot reduction) and enqueues nothing behind it
    # before every rank's producer is enqueued: a kernel queued behind a spinning one could hold up a producer sharing its queue.
    w_local = [torch.empty(n, device=DEV) for n in counts]  # an empty shard's tensor has no data pointer, as in the sharded generation
    torch.cuda.synchronize()
    for r, px in enumerate(world.px):
        lo, n = world.row0[r], counts[r]
        with world.on(r):
            px.rank_sharded(px.f_all[lo:lo + n], method, False, offsets, w_local[r])
    world.producers_done()
    sharded = []
    for r, px in enumerate(world.px):
        with world.on(r):
            summed = dist.partial_gradients(shards[r], w_local[r], world.row0[r], method, local_weights_of=N, peer=px)
            sharded.append(dist.finalize_gradients(summed, N))
    world.check(1, 1, f_written=False)  # no rank holds the other shards' fitnesses
    sharded = [{k: v.clone() for k, v in s.items()} for s in sharded]  # views of each rank's reduction buffer
    # the replicated path: the global ranking, sliced by partial_gradients
    w_all = ops.rank(f, method, False)
    torch.cuda.synchronize()
    replicated = []
    for r, px in enumerate(world.px):
        with world.on(r):
            replicated.append(dist.finalize_gradients(dist.partial_gradients(shards[r], w_all, world.row0[r], method, peer=px), N))
    world.check(1, 2, f_written=False)
    for r in range(world.R):
        for k in ("mu", "sigma"):
            assert same_bits(sharded[r][k], replicated[r][k]), (r, k)
            assert same_bits(sharded[r][k], sharded[0][k]), (r, k)
    whole = dist.compute_gradients(X, f, objective_sense="min", ranking_method=method)
    for k in ("mu", "sigma"):
        scale = float(whole[k].abs().max())
        torch.testing.assert_close(sharded[0][k], whole[k], rtol=1e-4, atol=1e-5 * scale)


# ------------------------------------------------------------------------------------------------ (f) argument errors
def test_peer_entry_points_reject_bad_arguments_without_launching():
    lib = nat.lib()
    world = SimWorld([8, 8], 4)
    px = world.px[0]
    mu, sigma = distribution_params(4, 1)
    w = torch.zeros(8, device=DEV)
    ws = torch.empty(lib.evok_grad_workspace_bytes(8, 4), dtype=torch.uint8, device=DEV)
    dst = torch.zeros(8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream

    def table(ptrs):
        return (ctypes.c_void_p * len(ptrs))(*ptrs)

    f17, flags17 = table([px.peer_f[0]] * 17), table([px.peer_flags_f[0]] * 17)
    slots17, gflags17 = table([px.peer_slots[0]] * 17), table([px.peer_flags_g[0]] * 17)
    null_f, null_flags = table([px.peer_f[0], None]), table([None, px.peer_flags_f[1]])
    null_slots, null_gflags = table([px.peer_slots[0], None]), table([None, px.peer_flags_g[1]])

    def sample_push(world_, rank, pf, pflags):
        return lib.evok_sample_eval_push(ops.OBJ_SPHERE, None, 0, mu.data_ptr(), sigma.data_ptr(), 0, 8, 4, 0, 1, 2, None, world_, rank, pf, pflags,
                                         px.epoch_f, px._counter(0), stream)

    def grad_push(world_, rank, pslots, pflags):
        return lib.evok_grad_push(ops.GRAD_SEPARABLE, None, 0, w.data_ptr(), mu.data_ptr(), sigma.data_ptr(), 0, 8, 4, 1, 2, None, 1.0, 1.0,
                                  world_, rank, pslots, pflags, px.epoch_g, px._counter(1), ws.data_ptr(), ws.numel(), stream)

    def peer_push(world_, rank, pf, pflags, n_bytes=32):
        return lib.evok_peer_push(px.f_all.data_ptr(), n_bytes, 0, world_, rank, pf, pflags, px.epoch_f, stream)

    calls = []
    for fn, tabs17, tabs in ((sample_push, (f17, flags17), (px.peer_f, px.peer_flags_f)),
                             (grad_push, (slots17, gflags17), (px.peer_slots, px.peer_flags_g)),
                             (peer_push, (f17, flags17), (px.peer_f, px.peer_flags_f))):
        calls += [(fn, (0, 0) + tabs, E_BADSIZE), (fn, (17, 0) + tabs17, E_BADSIZE), (fn, (2, 2) + tabs, E_BADSIZE), (fn, (2, -1) + tabs, E_BADSIZE)]
    calls += [(sample_push, (2, 0, null_f, px.peer_flags_f), E_NULLPTR), (sample_push, (2, 0, px.peer_f, null_flags), E_NULLPTR),
              (grad_push, (2, 0, null_slots, px.peer_flags_g), E_NULLPTR), (grad_push, (2, 0, px.peer_slots, null_gflags), E_NULLPTR),
              (peer_push, (2, 0, null_f, px.peer_flags_f), E_NULLPTR), (peer_push, (2, 0, px.peer_f, null_flags), E_NULLPTR),
              (peer_push, (2, 0, px.peer_f, px.peer_flags_f, 30), E_BADSIZE), (peer_push, (2, 0, px.peer_f, px.peer_flags_f, 2), E_BADSIZE)]
    for world_ in (0, 17):
        calls += [(lib.evok_peer_wait, (px._flags_f_ptr, world_, px.epoch_f, px._counter(3), TIMEOUT_NS, stream), E_BADSIZE),
                  (lib.evok_peer_reduce, (px.slots.data_ptr(), world_, 8, px._flags_g_ptr, px.epoch_g, px._counter(2), px._counter(3),
                                          TIMEOUT_NS, dst.data_ptr(), stream), E_BADSIZE)]
    calls += [(lib.evok_peer_wait, (None, 2, px.epoch_f, px._counter(3), TIMEOUT_NS, stream), E_NULLPTR),
              (lib.evok_peer_wait, (px._flags_f_ptr, 2, None, px._counter(3), TIMEOUT_NS, stream), E_NULLPTR),
              (lib.evok_peer_reduce, (None, 2, 8, px._flags_g_ptr, px.epoch_g, px._counter(2), px._counter(3), TIMEOUT_NS, dst.data_ptr(),
                                      stream), E_NULLPTR),
              (lib.evok_peer_reduce, (px.slots.data_ptr(), 2, 8, None, px.epoch_g, px._counter(2), px._counter(3), TIMEOUT_NS, dst.data_ptr(),
                                      stream), E_NULLPTR),
              (lib.evok_peer_reduce, (px.slots.data_ptr(), 2, 8, px._flags_g_ptr, px.epoch_g, px._counter(2), px._counter(3), TIMEOUT_NS, None,
                                      stream), E_NULLPTR)]
    before = lib.evok_launch_count()
    for fn, args, want in calls:
        assert fn(*args) == want, (getattr(fn, "__name__", fn), args[:2], want)
    assert lib.evok_launch_count() == before
    world.check(0, 0, f_written=False)
