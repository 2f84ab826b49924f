"""Restarts for the functional CMA-ES families: `restarts(state, ...) -> RestartState`, `restarts_tell(rs, values, evals)`.

A batch of `cmaes` or `sepcmaes` searches used as a multi-start global optimiser: every item keeps its best solution ever, checks
the termination criteria of Hansen's tutorial (The CMA Evolution Strategy: A Tutorial, appendix B.3) after each of its updates,
and starts again from a uniform centre in [lb, ub] with its initial step size when one fires.  Each item has its own generation
counter, which drives its h_sig and its decomposition schedule, so a restarted item runs exactly as a fresh search would.

    state = cmaes(center_init=torch.empty(1024, 10, device="cuda").uniform_(-5, 5), stdev_init=2.0, objective_sense="min")
    rs = restarts(state, lb=-5.0, ub=5.0)
    for _ in range(generations):
        values, evals = cmaes_ask_and_evaluate(rs.search, objective=rastrigin)
        rs = restarts_tell(rs, values, evals)
    rs.best_values, rs.best_evals, rs.num_restarts

On CUDA float32 a generation is the family's stages, with per-item counters in the update, and one restart stage (one launch;
two for the full family, whose second launch resets C and A of the restarted items): nothing is read back to the host.  With
decompose_C_freq > 1 the full family then factors C of every item in every generation and keeps the old factor where the item
is not due, since which items are due is only known on the device.  Anywhere else the same algorithm runs as batched torch ops.

`stop_flags` bits (ops.RESTART_CRITERIA): 0 tol_fun, 1 tol_x, 2 tol_x_up, 3 max_condition, 4 min_fitness_stdev, 5 max_generations,
6 non-finite state (always on), 7 small-run budget (BIPOP only, always on there: a small run has used half the evaluations of the
item's latest large run).

IPOP (Auger & Hansen, "A Restart CMA Evolution Strategy With Increasing Population Size", CEC 2005):
`restarts(state, ..., popsize_multiplier=2, max_popsize=640)` multiplies an item's population size at each of its restarts, along
the ladder lambda_0 = state.popsize, lambda_{k+1} = min(int(multiplier * lambda_k), max_popsize), with the default learning rates
of each size.  Items restart at different times, so the populations are padded: the ask draws max_popsize rows for every item
(`rs.search` has the top tier's popsize) and item b uses only its first `rs.popsize[b]` rows.  Its other rows are pad rows: their
values and evals may hold anything, NaN and inf included, and never reach the state, the best ever, the history or the criteria.
On the kernels the stages that depend on the population size read the item's tier from device tables: still no host reads.

BIPOP (Hansen, "Benchmarking a BI-Population CMA-ES on the BBOB-2009 Function Testbed", GECCO 2009 workshops):
`restarts(state, ..., popsize_multiplier=2, max_popsize=640, bipop=True)` interleaves two regimes per item.  Large runs climb IPOP's
ladder with the default step size; small runs draw a population size lambda_s = floor(lambda_0 (lambda_l / (2 lambda_0))^(u1^2))
(at least lambda_0; lambda_l the latest large run's) and a step size sigma_def 10^(-2 u2), and stop once they have used half the
evaluations of the latest large run (bit 7).  At each restart the regime that has used fewer evaluations runs next, large on a tie
(so the first restart is large); the first run counts in neither budget.  The tables hold the ladder's tiers and then one tier
per population size lambda_0 .. max(lambda_0, max_popsize // 2), so the small tier of lambda is n_large + lambda - lambda_0.
"""

from __future__ import annotations

import math
from typing import NamedTuple, Optional, Union

import torch

from ... import ops
from ..cmaes import CMAESHyperparameters, cmaes_hyperparameters
from . import funccmaes, funcsepcmaes
from .funccmaes import CMAESState, _host_float
from .funcsepcmaes import SepCMAESState
from .fused import LazyPopulation
from .misc import draw_philox_seed, on_kernels

MAX_TIERED_POPSIZE = 8192  # on the kernels: the largest padded population the one-launch counting rank takes


class IPOPLadder(NamedTuple):
    """The population sizes of an IPOP restart state and their constants: host values per tier k, and the device tables the
    tiered stages read at an item's tier."""
    popsizes: tuple  # lambda_k (host ints), increasing; the last is max_popsize
    history_lengths: tuple  # H_k = 10 + ceil(30 D / lambda_k) (host ints), decreasing
    hyperparameters: tuple  # CMAESHyperparameters of each tier
    counts: torch.Tensor  # (K,) int32: lambda_k
    history: torch.Tensor  # (K,) int64: H_k
    weights: torch.Tensor  # (K, max_popsize): the weights of tier k, zero past lambda_k
    consts: torch.Tensor  # (K, 10): the update constants of tier k (funccmaes.CONST_NAMES)
    decompose_C_freq: torch.Tensor  # (K,) int64
    # BIPOP (`bipop_ladder`): the number of ladder tiers; tiers n_large.. are the small runs' population sizes lambda_0, lambda_0 + 1,
    # .., and `hyperparameters` holds the ladder tiers' only (the small tiers' constants are in the tables).  None for IPOP.
    n_large: Optional[int] = None


class RestartState(NamedTuple):
    search: Union[CMAESState, SepCMAESState]  # the state to ask from
    best_values: torch.Tensor  # (..., D): the best solution ever per item, over all of its restarts (NaN until one was finite)
    best_evals: torch.Tensor  # (...): its fitness (+inf for "min", -inf for "max" until then)
    num_restarts: torch.Tensor  # (...) int64
    item_generation: torch.Tensor  # (...) int64: generations since the item's (re)start
    history: torch.Tensor  # (..., H): ring of the best fitness of the item's last H generations, slot (g - 1) % H for generation g
    stop_flags: torch.Tensor  # (...) int32: the criteria that fired in the last tell
    stdev_init: torch.Tensor  # (...): the step size an item restarts with
    lb: torch.Tensor  # (..., D)
    ub: torch.Tensor  # (..., D)
    tol_fun: Optional[float]
    tol_x: Optional[float]
    tol_x_up: Optional[float]
    max_condition: Optional[float]
    min_fitness_stdev: Optional[float]
    max_generations: Optional[float]
    # IPOP only (None otherwise); the history ring has H_0 slots, of which an item at tier k uses the first H_k
    tier: Optional[torch.Tensor] = None  # (...) int32: the item's rung of the ladder
    num_evaluations: Optional[torch.Tensor] = None  # (...) int64: the rows told to the item so far, lambda of its tier per tell
    ladder: Optional[IPOPLadder] = None
    # BIPOP only (None otherwise)
    regime: Optional[torch.Tensor] = None  # (...) int32: 0 the first run, 1 a large run, 2 a small run
    large_tier: Optional[torch.Tensor] = None  # (...) int32: the ladder rung of the item's latest large run (0 before any)
    large_evaluations: Optional[torch.Tensor] = None  # (...) int64: the rows told to the item in its large runs
    small_evaluations: Optional[torch.Tensor] = None  # (...) int64: in its small runs
    last_large_evaluations: Optional[torch.Tensor] = None  # (...) int64: in its latest large run (0 before one ended)
    run_stdev: Optional[torch.Tensor] = None  # (...): the step size the item's current run started with

    @property
    def thresholds(self) -> tuple:
        """The thresholds in the order of ops.RESTART_CRITERIA (None = off)."""
        return tuple(getattr(self, name) for name in ops.RESTART_CRITERIA)

    @property
    def popsize(self) -> torch.Tensor:
        """(...) the number of rows each item uses: lambda of its tier (a device gather), or the search's popsize."""
        if self.ladder is None:
            return torch.full(self.best_evals.shape, self.search.popsize, dtype=torch.int64, device=self.best_evals.device)
        return self.ladder.counts.long()[self.tier.long()]


def history_length(d: int, popsize: int) -> int:
    """H = 10 + ceil(30 D / popsize): the generations the tol_fun criterion looks back over."""
    return 10 + math.ceil(30 * d / popsize)


def _same_hyperparameters(a: CMAESHyperparameters, b: CMAESHyperparameters) -> bool:
    return all(torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y for x, y in zip(a, b))


def _make_hyperparameters(state: Union[CMAESState, SepCMAESState], limit: bool, device=None):
    """lambda -> the default hyperparameters of `state`'s family at population size lambda (on `device`, by default the state's)."""
    center = state.center
    sep, d = isinstance(state, SepCMAESState), center.shape[-1]
    dev = center.device if device is None else device
    return lambda lam: cmaes_hyperparameters(d, lam, dtype=center.dtype, device=dev, active=state.active, separable=sep, limit_C_decomposition=limit)


def _default_limit(state: Union[CMAESState, SepCMAESState]) -> Optional[bool]:
    """The limit_C_decomposition flag under which `state` has the default constants of its population size (None: neither)."""
    return next((lim for lim in (True, False) if _same_hyperparameters(_make_hyperparameters(state, lim)(state.popsize), state.hyperparameters)),
                None)


def ipop_ladder(state: Union[CMAESState, SepCMAESState], popsize_multiplier, max_popsize) -> IPOPLadder:
    """The IPOP ladder of `state` (see `restarts`).  Raises ValueError for a multiplier <= 1, a max_popsize below state.popsize, a
    step that does not grow, max_popsize > MAX_TIERED_POPSIZE on the kernels, and a state whose constants are not the defaults of
    its population size."""
    if max_popsize is None:
        raise ValueError("IPOP restarts need `max_popsize`, the population size the ladder stops at")
    mult = _host_float(popsize_multiplier, "popsize_multiplier")
    if not mult > 1.0:
        raise ValueError(f"`popsize_multiplier` must be > 1, got {mult}")
    lam0, cap = state.popsize, int(max_popsize)
    if cap < lam0:
        raise ValueError(f"`max_popsize` ({cap}) is below the search's popsize ({lam0})")
    sizes = [lam0]
    while sizes[-1] < cap:
        nxt = int(mult * sizes[-1])
        if nxt <= sizes[-1]:
            raise ValueError(f"popsize_multiplier {mult} does not grow the population size {sizes[-1]} (int({mult} * {sizes[-1]}) = {nxt})")
        sizes.append(min(nxt, cap))
    center = state.center
    if on_kernels(center) and cap > MAX_TIERED_POPSIZE:
        raise ValueError(f"`max_popsize` {cap} is above {MAX_TIERED_POPSIZE}, the largest padded population the kernels rank")
    d = center.shape[-1]
    limit = _default_limit(state)
    if limit is None:
        raise ValueError("IPOP uses the default learning rates of each population size: build the search with the default c_m and "
                         "learning-rate ratios")
    make = _make_hyperparameters(state, limit)
    hps = tuple(make(lam) for lam in sizes)
    K = len(sizes)
    weights = torch.zeros(K, cap, dtype=center.dtype, device=center.device)
    for k, hp in enumerate(hps):
        weights[k, :hp.popsize] = hp.weights
    hist = tuple(history_length(d, lam) for lam in sizes)
    dev = center.device
    return IPOPLadder(popsizes=tuple(sizes), history_lengths=hist, hyperparameters=hps, counts=torch.tensor(sizes, dtype=torch.int32, device=dev),
                      history=torch.tensor(hist, dtype=torch.int64, device=dev), weights=weights,
                      consts=torch.tensor([funccmaes._consts(hp) for hp in hps], dtype=center.dtype, device=dev),
                      decompose_C_freq=torch.tensor([hp.decompose_C_freq for hp in hps], dtype=torch.int64, device=dev))


def bipop_ladder(state: Union[CMAESState, SepCMAESState], popsize_multiplier, max_popsize) -> IPOPLadder:
    """The tables of BIPOP restarts of `state` (see `restarts`): the IPOP ladder (`ipop_ladder`, whose checks apply), then one
    small tier for every population size lambda_0 .. max(lambda_0, max_popsize // 2), with the default constants of that size.
    The small tiers' constants are computed on the host and copied to the state's device once: at max_popsize 8192 from
    lambda_0 = 10 the weight table has about 4100 x 8192 entries (134 MB in float32)."""
    lad = ipop_ladder(state, popsize_multiplier, max_popsize)
    lam0, cap, K = lad.popsizes[0], lad.popsizes[-1], len(lad.popsizes)
    small = tuple(range(lam0, max(lam0, cap // 2) + 1))
    center = state.center
    d, dev = center.shape[-1], center.device
    make = _make_hyperparameters(state, _default_limit(state), device="cpu")
    weights = torch.zeros(K + len(small), cap, dtype=center.dtype)
    weights[:K] = lad.weights.cpu()
    consts, freq = [], []
    for t, lam in enumerate(small):
        hp = make(lam)
        weights[K + t, :lam] = hp.weights
        consts.append(funccmaes._consts(hp))
        freq.append(hp.decompose_C_freq)
    hist = tuple(history_length(d, lam) for lam in small)
    return lad._replace(popsizes=lad.popsizes + small, history_lengths=lad.history_lengths + hist,
                        counts=torch.cat([lad.counts, torch.tensor(small, dtype=torch.int32, device=dev)]),
                        history=torch.cat([lad.history, torch.tensor(hist, dtype=torch.int64, device=dev)]), weights=weights.to(dev),
                        consts=torch.cat([lad.consts, torch.tensor(consts, dtype=center.dtype).to(dev)]),
                        decompose_C_freq=torch.cat([lad.decompose_C_freq, torch.tensor(freq, dtype=torch.int64, device=dev)]), n_large=K)


def restarts(state: Union[CMAESState, SepCMAESState], *, lb, ub, tol_fun: Optional[float] = 1e-12, tol_x: Optional[float] = 1e-12,
             tol_x_up: Optional[float] = 1e4, max_condition: Optional[float] = 1e14, min_fitness_stdev: Optional[float] = None,
             max_generations: Optional[int] = None, popsize_multiplier: Optional[float] = None, max_popsize: Optional[int] = None,
             bipop: bool = False) -> RestartState:
    """A restart state around `state` (a `CMAESState` or `SepCMAESState`).  `lb`, `ub`: the box the restarted centres are drawn
    from, scalars, (D,) or (..., D), finite with lb < ub.  A threshold of None turns its criterion off.  Every item's generation
    counter starts at `state.generation` and its restart step size is its current sigma.

    IPOP: with `popsize_multiplier` (> 1) and `max_popsize` (required with it), every item starts at tier 0, popsize
    lambda_0 = state.popsize, and each of its restarts moves it one tier up the ladder lambda_{k+1} = min(int(popsize_multiplier *
    lambda_k), max_popsize) (`ipop_ladder`), with the hyperparameters of `cmaes_hyperparameters` at that size.  `state` must have
    the default constants of its own size.  `rs.search` then asks for max_popsize rows per item (its popsize is the top tier's);
    item b uses the first `rs.popsize[b]` and ignores the others (pad rows, which may hold anything).  On the kernels
    max_popsize is at most 8192.

    BIPOP: with `bipop=True` as well (it needs `popsize_multiplier` and `max_popsize`, with the same checks), a restarted item runs
    either a large run one rung up the ladder or a small run of random population size in [lambda_0, max_popsize // 2] and step
    size in (sigma_def / 100, sigma_def] (sigma_def: the item's restart step size), whichever regime has used fewer evaluations
    (`bipop_ladder`; the module's docstring has the rule).  tol_x and tol_x_up then compare against the step size the current run
    started with (`rs.run_stdev`)."""
    if not isinstance(state, (CMAESState, SepCMAESState)):
        raise TypeError(f"`restarts` takes a CMAESState or a SepCMAESState, got {type(state).__name__}")
    center = state.center
    batch, d = tuple(center.shape[:-1]), center.shape[-1]
    bounds = []
    for name, v in (("lb", lb), ("ub", ub)):
        t = torch.as_tensor(v, dtype=center.dtype, device=center.device)
        try:
            t = t.expand(batch + (d,))
        except RuntimeError:
            raise ValueError(f"`{name}` of shape {tuple(t.shape)} does not broadcast to the search's {batch + (d,)}") from None
        bounds.append(t.contiguous().clone())
    lb_t, ub_t = bounds
    if not bool(torch.isfinite(lb_t).all() & torch.isfinite(ub_t).all() & (lb_t < ub_t).all()):
        raise ValueError("`lb` and `ub` must be finite with lb < ub")
    th = {}
    for name, v in (("tol_fun", tol_fun), ("tol_x", tol_x), ("tol_x_up", tol_x_up), ("max_condition", max_condition),
                    ("min_fitness_stdev", min_fitness_stdev), ("max_generations", max_generations)):
        th[name] = None if v is None else _host_float(v, name)
    maximize = state.maximize
    ladder = None
    if bipop and (popsize_multiplier is None or max_popsize is None):
        raise ValueError("BIPOP restarts climb an IPOP ladder in their large runs: give `popsize_multiplier` and `max_popsize` with `bipop`")
    if popsize_multiplier is not None or max_popsize is not None:
        if popsize_multiplier is None:
            raise ValueError("`max_popsize` is the cap of IPOP restarts: give `popsize_multiplier` with it")
        ladder = (bipop_ladder if bipop else ipop_ladder)(state, popsize_multiplier, max_popsize)
    H = history_length(d, state.popsize)
    opts = dict(dtype=center.dtype, device=center.device)
    zeros = lambda dt: torch.zeros(batch, dtype=dt, device=center.device)  # noqa: E731
    policy = {} if not bipop else dict(regime=zeros(torch.int32), large_tier=zeros(torch.int32), large_evaluations=zeros(torch.int64),
                                       small_evaluations=zeros(torch.int64), last_large_evaluations=zeros(torch.int64),
                                       run_stdev=state.sigma.clone())
    return RestartState(
        search=state if ladder is None else state._replace(hyperparameters=ladder.hyperparameters[-1]),
        best_values=torch.full(batch + (d,), math.nan, **opts),
        best_evals=torch.full(batch, -math.inf if maximize else math.inf, **opts),
        num_restarts=torch.zeros(batch, dtype=torch.int64, device=center.device),
        item_generation=torch.full(batch, state.generation, dtype=torch.int64, device=center.device),
        history=torch.full(batch + (H,), math.nan, **opts),
        stop_flags=torch.zeros(batch, dtype=torch.int32, device=center.device),
        stdev_init=state.sigma.clone(),
        lb=lb_t,
        ub=ub_t,
        **th,
        **({} if ladder is None else dict(tier=torch.zeros(batch, dtype=torch.int32, device=center.device),
                                          num_evaluations=torch.zeros(batch, dtype=torch.int64, device=center.device), ladder=ladder)),
        **policy,
    )


def restarts_tell(rs: RestartState, values: Union[torch.Tensor, LazyPopulation], evals: torch.Tensor) -> RestartState:
    """The family's tell with per-item generation counters, then per item: best ever, history, the criteria, and the re-initialisation
    of the items that met one.  `values` as the family's tell takes it (a separable search also takes the LazyPopulation that
    `sepcmaes_ask_and_evaluate(..., lazy=True)` returned).  `rs` is left unchanged.  IPOP: item b at tier k is told its first
    lambda_k rows with tier k's constants; its evaluations count grows by lambda_k, and a restart moves it to tier k + 1 (the top
    tier stays).  BIPOP: the same, with the regime's budget growing too and the regime policy choosing a restarted item's tier."""
    search = rs.search
    sep = isinstance(search, SepCMAESState)
    center = search.center
    batch, d = tuple(center.shape[:-1]), center.shape[-1]
    B, n = math.prod(batch), search.popsize
    family = funcsepcmaes if sep else funccmaes
    ipop = rs.ladder is not None
    tier = rs.tier.reshape(B).clone() if ipop else None
    new, steps = family._tell(search, values, evals, rs.item_generation.reshape(B), tiers=(rs.ladder, tier) if ipop else None)
    f = torch.as_tensor(evals, dtype=center.dtype, device=center.device).reshape(B, n)
    lazy = isinstance(values, LazyPopulation)
    x = None if lazy else torch.as_tensor(values, dtype=center.dtype, device=center.device).reshape(B, n, d)
    mat = (B, d) if sep else (B, d, d)
    st = dict(m=new.center.reshape(B, d), sigma=new.sigma.reshape(B), p_sigma=new.p_sigma.reshape(B, d), p_c=new.p_c.reshape(B, d),
              C=new.C.reshape(mat), A=new.A.reshape(mat), s=new.s.reshape(B, d) if sep else None)
    r = dict(history=rs.history.reshape(B, -1).clone(), best_x=rs.best_values.reshape(B, d).clone(), best_f=rs.best_evals.reshape(B).clone(),
             num_restarts=rs.num_restarts.reshape(B).clone())
    sigma0, lb, ub = rs.stdev_init.reshape(B), rs.lb.reshape(B, d), rs.ub.reshape(B, d)
    n_evals = rs.num_evaluations.reshape(B).clone() if ipop else None
    bipop = rs.regime is not None
    policy = {k: getattr(rs, k).reshape(B).clone() for k in BIPOP_FIELDS} if bipop else {}
    if lazy or on_kernels(center):
        # in place on the tell's fresh tensors and on the clones above
        flags = torch.empty(B, dtype=torch.int32, device=center.device)
        draw = dict(m_draw=search.center.reshape(B, d), s_draw=search.s.reshape(B, d), draw_seed=values.seed) if lazy else {}
        if ipop:
            draw.update(tier=tier, tier_counts=rs.ladder.counts, tier_history=rs.ladder.history, num_evaluations=n_evals)
        if bipop:
            draw.update(policy, n_large=rs.ladder.n_large, popsize0=rs.ladder.popsizes[0])
        ops.cma_restart_batched(sep, f.contiguous(), None if lazy else x.contiguous(), search.maximize, steps, st["m"], st["sigma"], st["p_sigma"],
                                st["p_c"], st["C"], st["A"], st["s"], r["history"], r["best_x"], r["best_f"], r["num_restarts"], flags,
                                sigma0.contiguous(), lb, ub, rs.thresholds, seed=draw_philox_seed(), **draw)
    else:
        if ipop:
            r.update(tier=tier, num_evaluations=n_evals, **policy)
        st, r, steps, flags = _restart_torch(rs.thresholds, sep, search.maximize, f, x, steps, st, r, sigma0, lb, ub, ladder=rs.ladder)
        if ipop:
            tier, n_evals = r["tier"], r["num_evaluations"]
            policy = {k: r[k] for k in policy}
    vec = batch + (d,)
    new = new._replace(center=st["m"].view(vec), sigma=st["sigma"].view(batch), p_sigma=st["p_sigma"].view(vec), p_c=st["p_c"].view(vec),
                       C=st["C"].view(vec if sep else vec + (d,)), A=st["A"].view(vec if sep else vec + (d,)),
                       **({"s": st["s"].view(vec)} if sep else {}))
    return rs._replace(search=new, best_values=r["best_x"].view(vec), best_evals=r["best_f"].view(batch), num_restarts=r["num_restarts"].view(batch),
                       item_generation=steps.view(batch), history=r["history"].view(batch + (-1,)), stop_flags=flags.view(batch),
                       **(dict(tier=tier.view(batch), num_evaluations=n_evals.view(batch)) if ipop else {}),
                       **{k: v.view(batch) for k, v in policy.items()})


BIPOP_FIELDS = ("regime", "large_tier", "large_evaluations", "small_evaluations", "last_large_evaluations", "run_stdev")


def _restart_torch(thresholds, sep, maximize, f, x, gen, st, r, sigma0, lb, ub, ladder=None) -> tuple:
    """The restart stage as batched torch ops (the semantics of evok_cma_restart_batched; the new centres from torch.rand(B, D)).
    With `ladder` (IPOP; r then also holds "tier" and "num_evaluations"), N and H of each item come from its tier, and the
    evaluation count and the tier advance follow (evok_cma_restart_batched_tiered).  With a BIPOP ladder (ladder.n_large set; r then
    also holds BIPOP_FIELDS), the regime policy of evok_cma_restart_batched_bipop replaces the tier advance; sigma0 is the default
    step size, and u1, u2 of a small run come from torch.rand(B, 2) after the centres."""
    B, n = f.shape
    d = lb.shape[-1]
    H = r["history"].shape[-1]
    nan = torch.tensor(math.nan, dtype=f.dtype, device=f.device)
    real = hreal = None
    if ladder is not None:
        t = r["tier"].long()
        n_b, H = ladder.counts.long()[t], ladder.history[t]
        real = torch.arange(n, device=f.device) < n_b[:, None]
        hreal = torch.arange(r["history"].shape[-1], device=f.device) < H[:, None]
    bipop = ladder is not None and ladder.n_large is not None
    run0 = r["run_stdev"] if bipop else sigma0  # the step size tol_x and tol_x_up compare against
    fin = torch.isfinite(f) if real is None else torch.isfinite(f) & real
    key = torch.where(fin, f, -math.inf if maximize else math.inf)
    idx = key.argmax(-1) if maximize else key.argmin(-1)  # the first of equal values: the lower row wins ties
    g_best = key.gather(-1, idx[:, None])[:, 0]
    has = fin.any(-1)
    improved = has & (g_best > r["best_f"] if maximize else g_best < r["best_f"])
    best_x = torch.where(improved[:, None], x[torch.arange(B), idx], r["best_x"])
    best_f = torch.where(improved, g_best, r["best_f"])
    slot = torch.remainder(gen - 1, H)
    written = r["history"].scatter(1, slot[:, None], torch.where(has, g_best, nan)[:, None])
    history = torch.where((gen >= 1)[:, None], written, r["history"])

    sig, m, p_sigma, p_c, C, A = st["sigma"], st["m"], st["p_sigma"], st["p_c"], st["C"], st["A"]
    c_diag = C if sep else torch.diagonal(C, dim1=-2, dim2=-1)
    r_diag = C if sep else torch.diagonal(A, dim1=-2, dim2=-1)
    nan_to = lambda t, v: torch.where(torch.isnan(t), v, t)  # noqa: E731 -- maxima and minima ignore NaN (fmaxf / fminf)
    max_pc = nan_to(p_c.abs(), 0.0).amax(-1).clamp_min(0.0)
    max_sd = nan_to(c_diag.sqrt(), 0.0).amax(-1).clamp_min(0.0)
    ratio = nan_to(r_diag, -math.inf).amax(-1) / nan_to(r_diag, math.inf).amin(-1)
    zero = torch.zeros(B, dtype=torch.bool, device=f.device)
    th = dict(zip(ops.RESTART_CRITERIA, thresholds))
    if real is None:
        f_all_fin, h_all_fin = fin.all(-1), torch.isfinite(history).all(-1)
        f_max, f_min, h_max, h_min = f.amax(-1), f.amin(-1), history.amax(-1), history.amin(-1)
        too_flat = zero if th["min_fitness_stdev"] is None or n < 2 else f.std(-1) < th["min_fitness_stdev"]
    else:  # only the first N_b values and H_b slots of each item
        f_all_fin, h_all_fin = (fin | ~real).all(-1), (torch.isfinite(history) | ~hreal).all(-1)
        f_max, f_min = torch.where(real, f, -math.inf).amax(-1), torch.where(real, f, math.inf).amin(-1)
        h_max, h_min = torch.where(hreal, history, -math.inf).amax(-1), torch.where(hreal, history, math.inf).amin(-1)
        too_flat = zero
        if th["min_fitness_stdev"] is not None:
            fr = torch.where(real, f, 0.0)
            mean = fr.sum(-1) / n_b
            var = torch.where(real, (fr - mean[:, None]) ** 2, 0.0).sum(-1) / (n_b - 1).clamp_min(1)
            too_flat = (n_b > 1) & (var.sqrt() < th["min_fitness_stdev"])
    bits = [
        zero if th["tol_fun"] is None else ((gen >= H) & f_all_fin & h_all_fin
                                            & (torch.maximum(f_max, h_max) - torch.minimum(f_min, h_min) < th["tol_fun"])),
        zero if th["tol_x"] is None else sig * torch.maximum(max_pc, max_sd) < th["tol_x"] * run0,
        zero if th["tol_x_up"] is None else sig * max_sd > th["tol_x_up"] * run0,
        zero if th["max_condition"] is None else (ratio if sep else ratio * ratio) > th["max_condition"],
        too_flat,
        zero if th["max_generations"] is None else gen >= th["max_generations"],
        ~(sig > 0) | ~torch.isfinite(sig) | ~torch.isfinite(torch.cat([m, p_sigma, p_c, c_diag], -1)).all(-1),
    ]
    if bipop:
        regime = r["regime"]
        n_large_ev = r["large_evaluations"] + torch.where(regime == 1, n_b, 0)
        n_small_ev = r["small_evaluations"] + torch.where(regime == 2, n_b, 0)
        bits.append((regime == 2) & (2 * gen * n_b >= r["last_large_evaluations"]))
    flags = sum(b.to(torch.int32) << k for k, b in enumerate(bits))
    go = flags != 0
    centre = lb + (ub - lb) * torch.rand(B, d, dtype=f.dtype, device=f.device)
    s0 = sigma0
    if bipop:
        policy = _bipop_policy(ladder, go, regime, gen, n_b, n_large_ev, n_small_ev, r, sigma0, torch.rand(B, 2, dtype=f.dtype, device=f.device))
        s0 = policy["run_stdev"]
    col = go[:, None]
    out = dict(m=torch.where(col, centre, m), sigma=torch.where(go, s0, sig), p_sigma=torch.where(col, 0.0, p_sigma), p_c=torch.where(col, 0.0, p_c))
    if sep:
        out.update(C=torch.where(col, 1.0, C), A=torch.where(col, 1.0, A), s=torch.where(col, s0[:, None].expand(B, d), st["s"]))
    else:
        eye = torch.eye(d, dtype=f.dtype, device=f.device)
        out.update(C=torch.where(go[:, None, None], eye, C), A=torch.where(go[:, None, None], eye, A), s=None)
    out_r = dict(history=torch.where(col, nan, history), best_x=best_x, best_f=best_f, num_restarts=r["num_restarts"] + go.to(torch.int64))
    if bipop:
        out_r.update(num_evaluations=r["num_evaluations"] + n_b, **policy)
    elif ladder is not None:
        out_r.update(num_evaluations=r["num_evaluations"] + n_b, tier=torch.where(go, torch.clamp_max(r["tier"] + 1, len(ladder.popsizes) - 1), r["tier"]))
    r = out_r
    return out, r, torch.where(go, 0, gen), flags


def _bipop_policy(ladder, go, regime, gen, n_b, n_large_ev, n_small_ev, r, sigma_def, u) -> dict:
    """The BIPOP fields after a tell, `go` the items that restart: the next run large (one rung up) when n_large_ev <= n_small_ev,
    else small, of population size max(lambda_0, floor(lambda_0 exp(u1^2 log(lambda_l / (2 lambda_0))))) and step size
    sigma_def 10^(-2 u2), in float64 (u (B, 2) in [0, 1))."""
    K, lam0 = ladder.n_large, ladder.popsizes[0]
    lt = r["large_tier"]
    large = n_large_ev <= n_small_ev
    last = torch.where(go & (regime == 1), gen * n_b, r["last_large_evaluations"])
    lt_up = torch.clamp_max(lt + 1, K - 1)
    u1, u2 = u[:, 0].double(), u[:, 1].double()
    lam_l = ladder.counts.long()[lt.long()].double()
    lam_s = torch.floor(lam0 * torch.exp(u1 * u1 * torch.log(0.5 * lam_l / lam0))).clamp_min(lam0).long()
    small_tier = torch.clamp_max(K + lam_s - lam0, len(ladder.popsizes) - 1).to(torch.int32)
    small_stdev = (sigma_def.double() * torch.pow(10.0, -2.0 * u2)).to(sigma_def.dtype)
    return dict(regime=torch.where(go, torch.where(large, 1, 2), regime).to(torch.int32),
                large_tier=torch.where(go & large, lt_up, lt).to(torch.int32),
                tier=torch.where(go, torch.where(large, lt_up, small_tier), r["tier"]).to(torch.int32),
                large_evaluations=n_large_ev, small_evaluations=n_small_ev, last_large_evaluations=last,
                run_stdev=torch.where(go, torch.where(large, sigma_def, small_stdev), r["run_stdev"]))
