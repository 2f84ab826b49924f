"""Tensor-level entry points of the sm_90a kernels (CUDA, fp32 only).

Each function validates its tensors, pulls raw pointers + the current stream and calls the C ABI of
libevok.so (include/evok.h).  Callers in this package decide *whether* a tensor goes to these kernels
(`uses_kernels`); there is no silent fallback from here: a missing library raises.
"""

from __future__ import annotations

import contextlib
import ctypes
import math
from typing import Optional

import torch

from . import _native as nat
from .tools.readonlytensor import as_plain_tensor

OBJ_NONE, OBJ_SPHERE, OBJ_RASTRIGIN, OBJ_ACKLEY = 0, 1, 2, 3
OBJ_USER_BASE = 64  # EVOK_OBJ_USER_BASE: the first id of an objective registered at run time (objectives.FusedObjective)
# name -> id; a FusedObjective adds its own name here
OBJECTIVE_IDS = {"sphere": OBJ_SPHERE, "rastrigin": OBJ_RASTRIGIN, "ackley": OBJ_ACKLEY}
RANK_IDS = {"centered": 0, "linear": 1, "nes": 2, "normalized": 3, "raw": 4}
GRAD_SEPARABLE, GRAD_SYMMETRIC, GRAD_EXP, GRAD_MOMENTS = 0, 1, 2, 3
NAN = float("nan")


# ------------------------------------------------------------------------------------------------ device-side kernel timers
# bench.py turns these on to time each kernel group with CUDA events recorded on the launching stream (no host sync while
# the generations run; the elapsed times are read after the timed region).
_timers: Optional[dict] = None


def enable_timers() -> None:
    global _timers
    _timers = {}


def disable_timers() -> None:
    global _timers
    _timers = None


class _timed:
    __slots__ = ("name", "start")

    def __init__(self, name: str):
        self.name = name

    def __enter__(self):
        if _timers is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.start.record()
        return self

    def __exit__(self, *exc):
        if _timers is not None:
            end = torch.cuda.Event(enable_timing=True)
            end.record()
            _timers.setdefault(self.name, []).append((self.start, end))
        return False


def timer_results() -> dict:
    """{kernel group: (launch count, mean milliseconds)}; call after torch.cuda.synchronize()."""
    out = {}
    for name, pairs in (_timers or {}).items():
        ms = [a.elapsed_time(b) for a, b in pairs]
        out[name] = (len(ms), sum(ms) / max(len(ms), 1))
    return out


_replayed_launches = 0


def count_replayed_launches(n: int) -> None:
    """CUDA-graph replays re-run captured kernels without passing through the library: the searchers report them here."""
    global _replayed_launches
    _replayed_launches += int(n)


def launch_count() -> int:
    """Kernels of libevok.so launched so far in this process: direct launches (counted inside the library) + graph replays."""
    return int(nat.lib().evok_launch_count()) + _replayed_launches


def uses_kernels(t: torch.Tensor) -> bool:
    """True for the tensors the hand-written kernels handle: CUDA + float32."""
    return t.is_cuda and t.dtype == torch.float32


def _vec(t: torch.Tensor, name: str, n: Optional[int] = None) -> torch.Tensor:
    if not (t.is_cuda and t.dtype == torch.float32 and t.ndim == 1 and t.is_contiguous()):
        raise ValueError(f"{name}: expected a contiguous 1-D float32 CUDA tensor, got {tuple(t.shape)} {t.dtype} {t.device}")
    if n is not None and t.numel() != n:
        raise ValueError(f"{name}: expected length {n}, got {t.numel()}")
    return as_plain_tensor(t)


def _mat(t: torch.Tensor, name: str) -> torch.Tensor:
    if not (t.is_cuda and t.dtype == torch.float32 and t.ndim == 2 and t.stride(1) == 1 and t.stride(0) >= t.shape[1]):
        raise ValueError(f"{name}: expected a row-major 2-D float32 CUDA tensor, got {tuple(t.shape)} strides {t.stride()} {t.dtype}")
    return as_plain_tensor(t)


def _ldx(X: Optional[torch.Tensor], n_rows: int, D: int) -> int:
    """Leading dimension of the optional population operand X (n_rows x D); 0 for X = None (nothing stored or read)."""
    if X is None:
        return 0
    _mat(X, "X")
    if X.shape != (n_rows, D):
        raise ValueError(f"X: expected shape {(n_rows, D)}, got {tuple(X.shape)}")
    return X.stride(0)


def _out_pair(mu: torch.Tensor, out_mu: Optional[torch.Tensor], out_sigma: Optional[torch.Tensor]) -> tuple:
    """The (mu, sigma) gradient outputs: the given D-vectors, or new ones."""
    D = mu.numel()
    return (torch.empty_like(mu) if out_mu is None else _vec(out_mu, "out_mu", D),
            torch.empty_like(mu) if out_sigma is None else _vec(out_sigma, "out_sigma", D))


def _check_scalar_sigma(sigma: torch.Tensor) -> None:
    if not (sigma.is_cuda and sigma.dtype == torch.float32 and sigma.numel() == 1):
        raise ValueError("sigma: expected a 1-element float32 CUDA tensor")


def _check_steps_dev(steps_dev: Optional[torch.Tensor]) -> None:
    if steps_dev is not None and not (steps_dev.is_cuda and steps_dev.dtype == torch.int64 and steps_dev.numel() == 1):
        raise ValueError("steps_dev: expected a 1-element int64 CUDA tensor")


def _host_floats(values, n: int):
    """The n host scalars `values` as a C float array (passed by pointer, read by the launch)."""
    vals = [float(v) for v in values]
    if len(vals) != n:
        raise ValueError(f"expected {n} host scalars, got {len(vals)}")
    return (ctypes.c_float * n)(*vals)


# ------------------------------------------------------------------------------------------------ K1 / K2
_loaded_objectives: set = set()
# the id of an objective with data (an instance of a registered objective) -> the device its data tensors are on
DATA_DEVICES: dict = {}


def _check_data_device(objective: int, t: torch.Tensor) -> None:
    if DATA_DEVICES.get(objective, t.device) != t.device:
        raise ValueError(f"the data of the objective is on {DATA_DEVICES[objective]}, the population on {t.device}")


def _load_objective(objective: int, t: torch.Tensor) -> None:
    """Load a registered objective's module on the device of `t` before its first launch there (evok_objective_load).  An
    objective with data evaluates only populations on the device of its data (ValueError)."""
    if objective < OBJ_USER_BASE:
        return
    _check_data_device(objective, t)
    key = (objective, t.device.index)
    if key not in _loaded_objectives:
        with torch.cuda.device(t.device):
            nat.check(nat.lib().evok_objective_load(objective), "evok_objective_load")
        _loaded_objectives.add(key)


def _offset_ptr(stream_offset: Optional[torch.Tensor]) -> Optional[int]:
    if stream_offset is None:
        return None
    if not (stream_offset.is_cuda and stream_offset.dtype == torch.int32 and stream_offset.numel() >= 1):
        raise ValueError("stream_offset: expected an int32 CUDA tensor with one element")
    return stream_offset.data_ptr()


def _sampler_args(objective: int, X, mu, sigma, n_rows: int, *, f=None, q=None, symmetric=False, row0=0, peer=None) -> Optional[int]:
    """The checks of `sample_eval`, `sample_eval_sq` (q) and `sample_eval_push` (peer) in their order, then `_load_objective`.
    Returns X's leading dimension, or None with no rows to sample (the push always launches: the peers wait for this rank's flag)."""
    D = mu.numel()
    _vec(mu, "mu"); _vec(sigma, "sigma", D)
    if q is not None:
        _vec(q, "q", n_rows)
    ldx = _ldx(X, n_rows, D)
    if peer is not None and row0 + n_rows > peer.popsize:
        raise ValueError("rows beyond the population the peer exchange was sized for")
    if q is not None and X is None and objective == OBJ_NONE:
        raise ValueError("X: the samples must be written somewhere when no objective is fused into the sampler")
    if f is not None:
        _vec(f, "f", n_rows)
    if peer is None and objective != OBJ_NONE and f is None:
        raise ValueError("f: a fitness buffer is required when an objective is fused into the sampler")
    if symmetric and (n_rows % 2 or row0 % 2):
        raise ValueError("symmetric sampling needs an even number of rows and an even first row")
    if peer is None and n_rows == 0:
        return None
    _load_objective(objective, mu)
    return ldx


def sample_eval(objective: int, X: Optional[torch.Tensor], mu: torch.Tensor, sigma: torch.Tensor, *, n_rows: int, symmetric: bool,
                seed: int, stream_id: int, row0: int = 0, f: Optional[torch.Tensor] = None,
                stream_offset: Optional[torch.Tensor] = None) -> None:
    if (ldx := _sampler_args(objective, X, mu, sigma, n_rows, f=f, symmetric=symmetric, row0=row0)) is None:
        return
    with _timed("sample_eval" if objective != OBJ_NONE else "sample"):
        rc = nat.lib().evok_sample_eval(objective, nat.ptr(X), ldx, mu.data_ptr(), sigma.data_ptr(), row0, n_rows, mu.numel(),
                                        int(symmetric), seed, stream_id, _offset_ptr(stream_offset), nat.ptr(f), nat.stream_of(mu))
    nat.check(rc, "evok_sample_eval")


def sample_eval_push(objective: int, X: Optional[torch.Tensor], mu: torch.Tensor, sigma: torch.Tensor, *, n_rows: int, symmetric: bool,
                     seed: int, stream_id: int, row0: int, peer, stream_offset: Optional[torch.Tensor] = None) -> None:
    """K1+K2 with the fitness all-gather fused in: row i's fitness lands in `f_all[row0 + i]` of every rank (`peer` is a
    evotorch_b200.peer.PeerExchange).  Follow with `peer.wait_fitness()` before reading `peer.f_all`."""
    ldx = _sampler_args(objective, X, mu, sigma, n_rows, row0=row0, peer=peer)
    with _timed("sample_eval"):
        rc = nat.lib().evok_sample_eval_push(objective, nat.ptr(X), ldx, mu.data_ptr(), sigma.data_ptr(), row0, n_rows, mu.numel(), int(symmetric),
                                             seed, stream_id, _offset_ptr(stream_offset), peer.world, peer.rank, peer.peer_f,
                                             peer.peer_flags_f, peer.epoch_f, peer._counter(0), nat.stream_of(mu))
    nat.check(rc, "evok_sample_eval_push")


def grad_push(form: int, X: Optional[torch.Tensor], w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, *, scale_mu: float,
              scale_sigma: float, peer, seed: int = 0, stream_id: int = 0, row0: int = 0, stream_offset: Optional[torch.Tensor] = None) -> None:
    """K4 with the send half of the gradient all-reduce fused in (X = None: regenerate the rows from the Philox counters).
    Follow with `peer.reduce_gradients()`."""
    _grad_call("evok_grad_push", "grad" if X is not None else "grad_regen", X, w, mu, sigma, None, lambda ldx, n, D, _: (
        form, nat.ptr(X), ldx, w.data_ptr(), mu.data_ptr(), sigma.data_ptr(), row0, n, D, seed, stream_id, _offset_ptr(stream_offset), scale_mu,
        scale_sigma, peer.world, peer.rank, peer.peer_slots, peer.peer_flags_g, peer.epoch_g, peer._counter(1)))


def evaluate(objective: int, X: torch.Tensor, f: Optional[torch.Tensor] = None) -> torch.Tensor:
    _mat(X, "X")
    n, D = X.shape
    if f is None:
        f = torch.empty(n, dtype=torch.float32, device=X.device)
    _vec(f, "f", n)
    _load_objective(objective, X)
    with _timed("eval"):
        rc = nat.lib().evok_eval(objective, X.data_ptr(), X.stride(0), n, D, f.data_ptr(), nat.stream_of(X))
    nat.check(rc, "evok_eval")
    return f


def evaluate_keyed(objective: int, X: torch.Tensor, *, seed: int, stream_id: int, row0: int = 0,
                   stream_offset: Optional[torch.Tensor] = None, f: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`evaluate` with the Philox draw of the rows (the keyword arguments of a `PhiloxDraw`): row i of X is global row row0 + i
    of the draw, so an objective with noise gives each row the noise the fused sampler gives it with the same draw.  For an
    objective without noise it is `evaluate`."""
    _mat(X, "X")
    n, D = X.shape
    if f is None:
        f = torch.empty(n, dtype=torch.float32, device=X.device)
    _vec(f, "f", n)
    _load_objective(objective, X)
    with _timed("eval"):
        rc = nat.lib().evok_eval_keyed(objective, X.data_ptr(), X.stride(0), row0, n, D, seed, stream_id, _offset_ptr(stream_offset),
                                       f.data_ptr(), nat.stream_of(X))
    nat.check(rc, "evok_eval_keyed")
    return f


def evaluate_batched(objective: int, X: torch.Tensor, *, seed: int, stream_id0: int = 0, f: Optional[torch.Tensor] = None) -> torch.Tensor:
    """K2 for a batch of populations in one launch: f[b, i] = objective(X[b, i]) for X (items, N, D) float32 CUDA with unit
    column stride (any item stride and row pitch), f (items, N).  Item b is evaluated as `evaluate_keyed(..., stream_id=stream_id0
    + b)` on its rows: an objective with noise draws row i of item b's noise from the draw (seed, stream_id0 + b), the noise the
    batched sampler gave row i of item b.  Per-item data of an instance is item b's.  A registered objective needs its batched
    evaluation kernels (`FusedObjective.compile_eval_batched`)."""
    if not (X.is_cuda and X.dtype == torch.float32 and X.ndim == 3 and (X.shape[2] <= 1 or X.stride(2) == 1)):
        raise ValueError(f"X: expected a float32 CUDA tensor of shape (items, N, D) with unit column stride, got {tuple(X.shape)} "
                         f"strides {X.stride()} {X.dtype} {X.device}")
    B, n, D = X.shape
    # the stride of a dimension of size 1 is arbitrary in torch: an item or row that has no successor needs none
    item_stride = X.stride(0) if B > 1 else 0
    ldx = X.stride(1) if n > 1 else D
    if f is None:
        f = torch.empty(B, n, dtype=torch.float32, device=X.device)
    f = _rows(f, "f", (B, n))
    _check_data_device(objective, X)
    if B == 0 or n == 0:  # nothing to evaluate (and an empty tensor may have no storage to point at)
        return f
    with _timed("eval"):
        rc = nat.lib().evok_eval_batched(objective, X.data_ptr(), item_stride, ldx, B, n, D, seed, stream_id0, f.data_ptr(), nat.stream_of(X))
    nat.check(rc, "evok_eval_batched")
    return f


def evaluate_transform_batched(objective: int, X: torch.Tensor, M: torch.Tensor, o: torch.Tensor, *, seed: int, stream_id0: int = 0,
                               f: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`evaluate_batched` of an objective with a transform (`jit.compile_transform`): its terms read y = M_b (x - o_b) of each row
    of item b.  M: (1 or items, D, D), o: (1 or items, D), float32 CUDA, each item's entries contiguous (1: shared by every item).
    Small D runs one fused launch; large D x - o, the batched 3xTF32 GEMM and the fold, with a workspace (`nat.workspace`)."""
    if not (X.is_cuda and X.dtype == torch.float32 and X.ndim == 3 and (X.shape[2] <= 1 or X.stride(2) == 1)):
        raise ValueError(f"X: expected a float32 CUDA tensor of shape (items, N, D) with unit column stride, got {tuple(X.shape)} "
                         f"strides {X.stride()} {X.dtype} {X.device}")
    B, n, D = X.shape
    for name, t, tail in (("M", M, (D, D)), ("o", o, (D,))):
        if not (t.dtype == torch.float32 and t.device == X.device and t.ndim == len(tail) + 1 and tuple(t.shape[1:]) == tail
                and t.shape[0] in (1, B) and t[0].is_contiguous()):
            raise ValueError(f"{name}: expected a float32 tensor of shape (1 or {B},) + {tail} on {X.device} with contiguous items, got "
                             f"{tuple(t.shape)} {t.dtype} {t.device}")
    sm = M.stride(0) if M.shape[0] > 1 else 0
    so = o.stride(0) if o.shape[0] > 1 else 0
    item_stride = X.stride(0) if B > 1 else 0
    ldx = X.stride(1) if n > 1 else D
    if f is None:
        f = torch.empty(B, n, dtype=torch.float32, device=X.device)
    f = _rows(f, "f", (B, n))
    _check_data_device(objective, X)
    if B == 0 or n == 0:
        return f
    lib = nat.lib()
    nbytes = lib.evok_eval_transform_workspace_bytes(M.data_ptr(), sm, B, n, D)
    ws = nat.workspace(X.device, nbytes, "transform") if nbytes else None
    with _timed("eval"):
        rc = lib.evok_eval_transform_batched(objective, X.data_ptr(), item_stride, ldx, M.data_ptr(), sm, o.data_ptr(), so, B, n, D, seed, stream_id0,
                                             nat.ptr(ws), nbytes, f.data_ptr(), nat.stream_of(X))
    nat.check(rc, "evok_eval_transform_batched")
    return f


# ------------------------------------------------------------------------------------------------ K3
def _rank_ws(device: torch.device, n: int) -> torch.Tensor:
    return nat.workspace(device, nat.lib().evok_rank_workspace_bytes(n), "rank")


def _rank_call(entry: str, keys: torch.Tensor, *args, timed: bool = True) -> None:
    """`entry`(*args, workspace, its size, stream) for a K3 entry point that sorts `keys`, timed as "rank" if `timed`."""
    ws = _rank_ws(keys.device, keys.shape[-1])
    with _timed("rank") if timed else contextlib.nullcontext():
        rc = getattr(nat.lib(), entry)(*args, ws.data_ptr(), ws.numel(), nat.stream_of(keys))
    nat.check(rc, entry)


def rank(f: torch.Tensor, method: str, higher_is_better: bool, out: Optional[torch.Tensor] = None,
         perm: Optional[torch.Tensor] = None) -> torch.Tensor:
    f = _vec(f, "fitnesses")
    n = f.numel()
    w = torch.empty_like(f) if out is None else _vec(out, "out", n)
    if perm is not None and not (perm.is_cuda and perm.dtype == torch.int64 and perm.is_contiguous() and perm.numel() == n):
        raise ValueError("perm: expected a contiguous int64 CUDA tensor of the same length")
    _rank_call("evok_rank", f, RANK_IDS[method], f.data_ptr(), n, int(bool(higher_is_better)), w.data_ptr(), nat.ptr(perm))
    return w


def argsort(keys: torch.Tensor, descending: bool) -> torch.Tensor:
    keys = _vec(keys, "keys")
    perm = torch.empty(keys.numel(), dtype=torch.int64, device=keys.device)
    _rank_call("evok_argsort", keys, keys.data_ptr(), keys.numel(), int(bool(descending)), perm.data_ptr(), timed=False)
    return perm


def rank_table(keys: torch.Tensor, descending: bool, table: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[i] = table[position of keys[i] in the stable sorted order] (position 0 = largest key if `descending`)."""
    keys = _vec(keys, "keys")
    n = keys.numel()
    _vec(table, "table", n)
    out = torch.empty_like(keys) if out is None else _vec(out, "out", n)
    _rank_call("evok_rank_table", keys, keys.data_ptr(), n, int(bool(descending)), table.data_ptr(), out.data_ptr())
    return out


def cmaes_row_weights(assigned: torch.Tensor, Z: torch.Tensor, active: bool, w_pos: torch.Tensor, w_act: torch.Tensor) -> None:
    """w_pos = max(assigned, 0); w_act = assigned > 0 ? assigned : D * assigned / ||z_i||^2 (or `assigned` when not `active`)."""
    _mat(Z, "Z")
    n, d = Z.shape
    _vec(assigned, "assigned", n); _vec(w_pos, "w_pos", n); _vec(w_act, "w_act", n)
    nat.check(nat.lib().evok_cmaes_row_weights(assigned.data_ptr(), Z.data_ptr(), Z.stride(0), n, d, int(bool(active)), w_pos.data_ptr(),
                                               w_act.data_ptr(), nat.stream_of(Z)), "evok_cmaes_row_weights")


def cmaes_vector_update(local_disp: torch.Tensor, shaped_disp: torch.Tensor, m: torch.Tensor, p_sigma: torch.Tensor, p_c: torch.Tensor,
                        sigma: torch.Tensor, consts, csa_squared: bool, k_out: torch.Tensor, *, steps: int = 0,
                        steps_dev: Optional[torch.Tensor] = None, h_sig_out: Optional[torch.Tensor] = None) -> None:
    """In place: m, p_sigma, sigma (1-element tensor), p_c; k_out (3 floats) = coefficients of the covariance update."""
    d = m.numel()
    _vec(local_disp, "local_disp", d); _vec(shaped_disp, "shaped_disp", d); _vec(m, "m"); _vec(p_sigma, "p_sigma", d); _vec(p_c, "p_c", d)
    _vec(k_out, "k_out", 3)
    _check_scalar_sigma(sigma)
    _check_steps_dev(steps_dev)
    nat.check(nat.lib().evok_cmaes_vector_update(local_disp.data_ptr(), shaped_disp.data_ptr(), d, m.data_ptr(), p_sigma.data_ptr(), p_c.data_ptr(),
                                                 sigma.data_ptr(), nat.ptr(steps_dev), int(steps), _host_floats(consts, 10), int(bool(csa_squared)),
                                                 k_out.data_ptr(), nat.ptr(h_sig_out), nat.stream_of(m)), "evok_cmaes_vector_update")


def sample_eval_sq(objective: int, X: Optional[torch.Tensor], mu: torch.Tensor, sigma: torch.Tensor, q: torch.Tensor, *, n_rows: int,
                   seed: int, stream_id: int, row0: int = 0, f: Optional[torch.Tensor] = None,
                   stream_offset: Optional[torch.Tensor] = None) -> None:
    """`sample_eval` (non-symmetric) that also writes q[i] = ||z_i||^2 of the unscaled normals; X / f are the same bits as
    `sample_eval` with the same arguments.  X = None: lazy population (needs an objective with a fused kernel)."""
    if (ldx := _sampler_args(objective, X, mu, sigma, n_rows, f=f, q=q)) is None:
        return
    with _timed("sepcma_sample"):
        rc = nat.lib().evok_sample_eval_sq(objective, nat.ptr(X), ldx, mu.data_ptr(), sigma.data_ptr(), row0, n_rows, mu.numel(), seed, stream_id,
                                           _offset_ptr(stream_offset), nat.ptr(f), q.data_ptr(), nat.stream_of(mu))
    nat.check(rc, "evok_sample_eval_sq")


def sepcma_moments(aw: torch.Tensor, q: Optional[torch.Tensor], active: bool, D: int, *, seed: int, stream_id: int, row0: int = 0,
                   stream_offset: Optional[torch.Tensor] = None, local: Optional[torch.Tensor] = None, S2: Optional[torch.Tensor] = None,
                   wsum: Optional[torch.Tensor] = None) -> tuple:
    """Separable CMA-ES moments over the population that `sample_eval_sq` drew with the same (seed, stream_id, row0, stream_offset),
    regenerated from Philox: local = sum_i a_i z_i, S2 = sum_i b_i z_i^2, wsum = sum_i b_i (1 element), with a_i = max(aw_i, 0) and
    b_i = aw_i, or with `active` b_i = aw_i > 0 ? aw_i : D aw_i / q_i.  Returns (local, S2, wsum)."""
    n = aw.numel()
    _vec(aw, "aw")
    if active:
        if q is None:
            raise ValueError("q: the squared norms are required with active weights")
        _vec(q, "q", n)
    dev = aw.device
    local = torch.empty(D, dtype=torch.float32, device=dev) if local is None else _vec(local, "local", D)
    S2 = torch.empty(D, dtype=torch.float32, device=dev) if S2 is None else _vec(S2, "S2", D)
    wsum = torch.empty(1, dtype=torch.float32, device=dev) if wsum is None else _vec(wsum, "wsum", 1)
    ws = nat.workspace(dev, nat.lib().evok_sepcma_workspace_bytes(n, D), "grad")
    with _timed("sepcma_moments"):
        rc = nat.lib().evok_sepcma_moments(aw.data_ptr(), nat.ptr(q), int(bool(active)), row0, n, D, seed, stream_id,
                                           _offset_ptr(stream_offset), local.data_ptr(), S2.data_ptr(), wsum.data_ptr(), ws.data_ptr(),
                                           ws.numel(), nat.stream_of(aw))
    nat.check(rc, "evok_sepcma_moments")
    return local, S2, wsum


def sepcma_update(local: torch.Tensor, S2: torch.Tensor, wsum: torch.Tensor, m: torch.Tensor, p_sigma: torch.Tensor, p_c: torch.Tensor,
                  sigma: torch.Tensor, C: torch.Tensor, A: torch.Tensor, s: torch.Tensor, consts, csa_squared: bool, *, decompose_C_freq: int,
                  steps: int = 0, steps_dev: Optional[torch.Tensor] = None, stdev_min: Optional[float] = None, stdev_max: Optional[float] = None,
                  m_prev: Optional[torch.Tensor] = None, s_prev: Optional[torch.Tensor] = None, h_sig_out: Optional[torch.Tensor] = None) -> None:
    """In place, one kernel: m, p_sigma, sigma (1-element tensor), p_c, C, A (diagonal, D-vectors) and s = sigma * A after one separable
    CMA-ES generation with the given moments (see `sepcma_moments`).  `consts` as for `cmaes_vector_update`.  m_prev / s_prev receive
    m and s from before the update."""
    d = m.numel()
    _vec(local, "local", d); _vec(S2, "S2", d); _vec(wsum, "wsum", 1); _vec(m, "m"); _vec(p_sigma, "p_sigma", d); _vec(p_c, "p_c", d)
    _vec(C, "C", d); _vec(A, "A", d); _vec(s, "s", d)
    for t, name in ((m_prev, "m_prev"), (s_prev, "s_prev")):
        if t is not None:
            _vec(t, name, d)
    _check_scalar_sigma(sigma)
    _check_steps_dev(steps_dev)
    if int(decompose_C_freq) < 1:
        raise ValueError("decompose_C_freq: expected a positive integer")
    lo = NAN if stdev_min is None else float(stdev_min)
    hi = NAN if stdev_max is None else float(stdev_max)
    with _timed("sepcma_update"):
        rc = nat.lib().evok_sepcma_update(local.data_ptr(), S2.data_ptr(), wsum.data_ptr(), d, m.data_ptr(), p_sigma.data_ptr(), p_c.data_ptr(),
                                          sigma.data_ptr(), C.data_ptr(), A.data_ptr(), s.data_ptr(), nat.ptr(m_prev), nat.ptr(s_prev),
                                          nat.ptr(steps_dev), int(steps), _host_floats(consts, 10), int(bool(csa_squared)),
                                          int(decompose_C_freq), lo, hi, nat.ptr(h_sig_out), nat.stream_of(m))
    nat.check(rc, "evok_sepcma_update")


def weights_adjust_(w: torch.Tensor, mode: int) -> torch.Tensor:
    _vec(w, "weights")
    nat.check(nat.lib().evok_weights_adjust(w.data_ptr(), w.numel(), mode, nat.stream_of(w)), "evok_weights_adjust")
    return w


def elite_mask(w: torch.Tensor, num_elites: int) -> torch.Tensor:
    w = _vec(w, "weights")
    mask = torch.empty_like(w)
    _rank_call("evok_elite_mask", w, w.data_ptr(), w.numel(), num_elites, mask.data_ptr(), timed=False)
    return mask


# ------------------------------------------------------------------------------------------------ K4
def _grad_call(entry: str, group: str, X: Optional[torch.Tensor], w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, outs, args):
    """The part of `grad`, `grad_regen`, `grad_hybrid` and `grad_push` they share: the checks of the samples X (n x D) when given,
    else n = len(w) and D = len(mu), then of w, mu and sigma against them; the outputs of `_out_pair(mu, *outs)` (`outs` None: the
    push writes none); then `entry`(*args(ldx, n, D, outputs), workspace, its size, stream) on X's device and stream (mu's without
    X), timed as `group`.  Returns the outputs."""
    if X is not None:
        _mat(X, "samples")
        n, D = X.shape
    else:
        n, D = w.numel(), mu.numel()
    _vec(w, "weights", n); _vec(mu, "mu", D); _vec(sigma, "sigma", D)
    on = mu if X is None else X
    out = None if outs is None else _out_pair(mu, *outs)
    ws = nat.workspace(on.device, nat.lib().evok_grad_workspace_bytes(n, D), "grad")
    with _timed(group):
        rc = getattr(nat.lib(), entry)(*args(0 if X is None else X.stride(0), n, D, out), ws.data_ptr(), ws.numel(), nat.stream_of(on))
    nat.check(rc, entry)
    return out


def grad(form: int, X: torch.Tensor, w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, scale_mu: float, scale_sigma: float,
         out_mu: Optional[torch.Tensor] = None, out_sigma: Optional[torch.Tensor] = None) -> tuple:
    return _grad_call("evok_grad", "grad", X, w, mu, sigma, (out_mu, out_sigma), lambda ldx, n, D, out: (
        form, X.data_ptr(), ldx, w.data_ptr(), mu.data_ptr(), sigma.data_ptr(), n, D, scale_mu, scale_sigma, out[0].data_ptr(), out[1].data_ptr()))


def grad_regen(form: int, w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, *, seed: int, stream_id: int, row0: int,
               scale_mu: float, scale_sigma: float, out_mu: Optional[torch.Tensor] = None,
               out_sigma: Optional[torch.Tensor] = None, stream_offset: Optional[torch.Tensor] = None) -> tuple:
    return _grad_call("evok_grad_regen", "grad_regen", None, w, mu, sigma, (out_mu, out_sigma), lambda ldx, n, D, out: (
        form, w.data_ptr(), mu.data_ptr(), sigma.data_ptr(), row0, n, D, seed, stream_id, _offset_ptr(stream_offset), scale_mu, scale_sigma,
        out[0].data_ptr(), out[1].data_ptr()))


GRAD_SPLIT_PERIOD = 16  # `split` of grad_hybrid counts rebuilt row groups per this many


def grad_hybrid(form: int, X: torch.Tensor, w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, *, seed: int, stream_id: int, row0: int,
                scale_mu: float, scale_sigma: float, split: int = -1, out_mu: Optional[torch.Tensor] = None,
                out_sigma: Optional[torch.Tensor] = None, stream_offset: Optional[torch.Tensor] = None) -> tuple:
    """`grad` over an X that `sample_eval` wrote from this very `mu` / `sigma` with the same seed, stream_id, row0 and
    stream_offset: `split` of every GRAD_SPLIT_PERIOD row groups are rebuilt from their Philox counters instead of being read
    (-1 = the library's choice).  Bit-identical to `grad(form, X, ...)` for every split."""
    if not -1 <= split <= GRAD_SPLIT_PERIOD:
        raise ValueError(f"split: expected -1 .. {GRAD_SPLIT_PERIOD}, got {split}")
    return _grad_call("evok_grad_hybrid", "grad_hybrid", X, w, mu, sigma, (out_mu, out_sigma), lambda ldx, n, D, out: (
        form, X.data_ptr(), ldx, w.data_ptr(), mu.data_ptr(), sigma.data_ptr(), row0, n, D, seed, stream_id, _offset_ptr(stream_offset),
        int(split), scale_mu, scale_sigma, out[0].data_ptr(), out[1].data_ptr()))


# ------------------------------------------------------------------------------------------------ K5
def clipup_step(g: torch.Tensor, velocity: torch.Tensor, stepsize: float, momentum: float, max_speed: float,
                step_out: Optional[torch.Tensor] = None, mu: Optional[torch.Tensor] = None) -> None:
    D = g.numel()
    _vec(g, "g"); _vec(velocity, "velocity", D)
    with _timed("mu_step"):
        rc = nat.lib().evok_clipup_step(g.data_ptr(), D, velocity.data_ptr(), stepsize, momentum, max_speed, nat.ptr(step_out),
                                        nat.ptr(mu), nat.stream_of(g))
    nat.check(rc, "evok_clipup_step")


def adam_step(g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, t: int, lr: float, beta1: float, beta2: float, eps: float,
              step_out: Optional[torch.Tensor] = None, mu: Optional[torch.Tensor] = None) -> None:
    D = g.numel()
    _vec(g, "g"); _vec(m, "m", D); _vec(v, "v", D)
    rc = nat.lib().evok_adam_step(g.data_ptr(), D, m.data_ptr(), v.data_ptr(), t, lr, beta1, beta2, eps, nat.ptr(step_out), nat.ptr(mu),
                                  nat.stream_of(g))
    nat.check(rc, "evok_adam_step")


def sgd_step(g: torch.Tensor, buf: Optional[torch.Tensor], first_step: bool, lr: float, momentum: float,
             step_out: Optional[torch.Tensor] = None, mu: Optional[torch.Tensor] = None) -> None:
    D = g.numel()
    _vec(g, "g")
    rc = nat.lib().evok_sgd_step(g.data_ptr(), D, nat.ptr(buf), int(first_step), lr, momentum, nat.ptr(step_out), nat.ptr(mu),
                                 nat.stream_of(g))
    nat.check(rc, "evok_sgd_step")


def axpy_(mu: torch.Tensor, g: torch.Tensor, lr: float) -> None:
    D = g.numel()
    _vec(g, "g"); _vec(mu, "mu", D)
    nat.check(nat.lib().evok_axpy(g.data_ptr(), D, lr, mu.data_ptr(), nat.stream_of(g)), "evok_axpy")


def _bound(x, D: int, device) -> tuple:
    """(vector pointer or None, scalar) for a None / scalar / vector bound."""
    if x is None:
        return None, NAN
    if isinstance(x, torch.Tensor) and x.ndim >= 1 and x.numel() > 1:
        v = x.to(device=device, dtype=torch.float32).contiguous()
        if v.numel() != D:
            raise IndexError(f"bound vector has length {v.numel()}, expected {D}")
        return v, NAN
    return None, float(x)


def sigma_update_(sigma: torch.Tensor, g: torch.Tensor, lr: float, exp_form: bool, lb=None, ub=None, max_change=None) -> None:
    D = sigma.numel()
    _vec(sigma, "sigma"); _vec(g, "g", D)
    lbv, lbs = _bound(lb, D, sigma.device)
    ubv, ubs = _bound(ub, D, sigma.device)
    mcv, mcs = _bound(max_change, D, sigma.device)
    with _timed("sigma_step"):
        rc = nat.lib().evok_sigma_update(sigma.data_ptr(), g.data_ptr(), D, lr, int(exp_form), nat.ptr(lbv), lbs, nat.ptr(ubv), ubs,
                                         nat.ptr(mcv), mcs, nat.stream_of(sigma))
    nat.check(rc, "evok_sigma_update")


def cem_finalize(s1: torch.Tensor, s2: torch.Tensor, sigma: torch.Tensor, num_elites: int) -> tuple:
    D = sigma.numel()
    gm, gs = torch.empty_like(sigma), torch.empty_like(sigma)
    nat.check(nat.lib().evok_cem_finalize(s1.data_ptr(), s2.data_ptr(), sigma.data_ptr(), D, num_elites, gm.data_ptr(), gs.data_ptr(),
                                          nat.stream_of(sigma)), "evok_cem_finalize")
    return gm, gs


# ------------------------------------------------------------------------------------------------ batched searches (functional API)
def _items(t: torch.Tensor, core_shape: tuple, name: str) -> tuple:
    """(tensor, n_items or None, item stride in elements) of an operand that is either shared (shape == core_shape, stride 0) or
    contiguous [items, *core_shape]."""
    if not (t.is_cuda and t.dtype == torch.float32):
        raise ValueError(f"{name}: expected a float32 CUDA tensor")
    t = as_plain_tensor(t)
    if tuple(t.shape) == tuple(core_shape):
        return t.contiguous(), None, 0
    if tuple(t.shape[1:]) != tuple(core_shape) or t.ndim != len(core_shape) + 1:
        raise ValueError(f"{name}: expected shape {core_shape} or (items, {', '.join(map(str, core_shape))}), got {tuple(t.shape)}")
    t = t.contiguous()
    return t, t.shape[0], int(t.stride(0))


def _rows(t: torch.Tensor, name: str, shape: tuple) -> torch.Tensor:
    """A 2-D operand of the batched stages: contiguous float32 CUDA of shape (items, n)."""
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape):
        raise ValueError(f"{name}: expected a contiguous float32 CUDA tensor of shape {shape}")
    return as_plain_tensor(t)


def sample_batched(out: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, *, symmetric: bool, seed: int, stream_id0: int = 0) -> torch.Tensor:
    """out[b] ~ N(mu[b], diag(sigma[b]^2)) for every batch item in one launch; item b uses Philox stream stream_id0 + b."""
    if not (out.is_cuda and out.dtype == torch.float32 and out.ndim == 3 and out.is_contiguous()):
        raise ValueError("out: expected a contiguous float32 CUDA tensor of shape (items, popsize, D)")
    B, n, d = out.shape
    mu, bm, sm = _items(mu, (d,), "mu")
    sigma, bs, ss = _items(sigma, (d,), "sigma")
    for cnt in (bm, bs):
        if cnt is not None and cnt != B:
            raise ValueError("mu / sigma: number of items differs from out")
    if symmetric and n % 2:
        raise ValueError(f"Symmetric sampling cannot be done if the number of solutions is odd: {n}")
    with _timed("sample"):
        rc = nat.lib().evok_sample_batched(out.data_ptr(), n * d, d, mu.data_ptr(), sm, sigma.data_ptr(), ss, B, n, d, int(symmetric),
                                           seed, stream_id0, nat.stream_of(out))
    nat.check(rc, "evok_sample_batched")
    return out


def sample_eval_batched(objective: int, X: Optional[torch.Tensor], mu: torch.Tensor, sigma: torch.Tensor, f: torch.Tensor, *, symmetric: bool,
                        seed: int, stream_id0: int = 0) -> torch.Tensor:
    """K1+K2 for every batch item in one launch: item b samples with Philox stream stream_id0 + b into X[b] (X = None: a lazy
    population, evaluated and not stored) and writes its fitnesses to f[b].  X: (items, N, D) or None, f: (items, N), mu / sigma:
    (D,) or (items, D).  Per item, X and f are the bits of `sample_eval(..., stream_id=stream_id0 + b)`.  A registered objective
    needs its batched kernels (`FusedObjective.compile_batched`)."""
    if objective == OBJ_NONE:
        raise ValueError("objective: EVOK_OBJ_NONE only samples; use sample_batched")
    if not (f.is_cuda and f.dtype == torch.float32 and f.ndim == 2):
        raise ValueError("f: expected a contiguous float32 CUDA tensor of shape (items, popsize)")
    B, n = f.shape
    d = mu.shape[-1]
    f = _rows(f, "f", (B, n))
    if X is not None:
        if not (X.is_cuda and X.dtype == torch.float32 and X.is_contiguous() and tuple(X.shape) == (B, n, d)):
            raise ValueError(f"X: expected a contiguous float32 CUDA tensor of shape {(B, n, d)}")
        X = as_plain_tensor(X)
    mu, bm, sm = _items(mu, (d,), "mu")
    sigma, bs, ss = _items(sigma, (d,), "sigma")
    for cnt in (bm, bs):
        if cnt is not None and cnt != B:
            raise ValueError("mu / sigma: number of items differs from f")
    _check_data_device(objective, f)
    if symmetric and n % 2:
        raise ValueError(f"Symmetric sampling cannot be done if the number of solutions is odd: {n}")
    with _timed("sample_eval"):
        rc = nat.lib().evok_sample_eval_batched(objective, nat.ptr(X), n * d, d, mu.data_ptr(), sm, sigma.data_ptr(), ss, B, n, d, int(symmetric),
                                                seed, stream_id0, f.data_ptr(), nat.stream_of(f))
    nat.check(rc, "evok_sample_eval_batched")
    return f


def rank_batched(f: torch.Tensor, method: str, higher_is_better: bool) -> torch.Tensor:
    """Utilities of `items` independent fitness vectors, f: (items, N)."""
    if not (f.is_cuda and f.dtype == torch.float32 and f.ndim == 2):
        raise ValueError("f: expected a float32 CUDA tensor of shape (items, N)")
    f = as_plain_tensor(f).contiguous()
    B, n = f.shape
    w = torch.empty_like(f)
    lib = nat.lib()
    ws = nat.workspace(f.device, max(lib.evok_rank_workspace_bytes(n), 8 * B + 256), "rank")
    with _timed("rank"):
        rc = lib.evok_rank_batched(RANK_IDS[method], f.data_ptr(), n, B, int(bool(higher_is_better)), w.data_ptr(), ws.data_ptr(), ws.numel(),
                                   nat.stream_of(f))
    nat.check(rc, "evok_rank_batched")
    return w


def elite_mask_batched(w: torch.Tensor, num_elites: int) -> torch.Tensor:
    B, n = w.shape
    w = _rows(w, "weights", (B, n))
    mask = torch.empty_like(w)
    _rank_call("evok_elite_mask_batched", w, w.data_ptr(), n, B, num_elites, mask.data_ptr(), timed=False)
    return mask


def weights_adjust_batched_(w: torch.Tensor, mode: int) -> torch.Tensor:
    B, n = w.shape
    _rows(w, "weights", (B, n))
    nat.check(nat.lib().evok_weights_adjust_batched(w.data_ptr(), n, B, mode, nat.stream_of(w)), "evok_weights_adjust_batched")
    return w


def _grad_batched_call(entry: str, group: str, w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, B: int, n: int, d: int, args) -> tuple:
    """The checks of `grad_batched` and `grad_batched_regen` (w: (B, n), mu / sigma: (d,) or (B, d)), then
    `entry`(*args(mu, item stride of mu, sigma, item stride of sigma), outputs, workspace, its size, stream) timed as `group`."""
    w = _rows(w, "w", (B, n))
    mu, bm, sm = _items(mu, (d,), "mu")
    sigma, bs, ss = _items(sigma, (d,), "sigma")
    for cnt in (bm, bs):
        if cnt is not None and cnt != B:
            raise ValueError("mu / sigma: number of items differs from w")
    out_mu = torch.empty(B, d, dtype=torch.float32, device=w.device)
    out_sigma = torch.empty_like(out_mu)
    lib = nat.lib()
    ws = nat.workspace(w.device, lib.evok_grad_batched_workspace_bytes(B, n, d), "grad_batched")
    with _timed(group):
        rc = getattr(lib, entry)(*args(mu, sm, sigma, ss), out_mu.data_ptr(), out_sigma.data_ptr(), ws.data_ptr(), ws.numel(), nat.stream_of(w))
    nat.check(rc, entry)
    return out_mu, out_sigma


def grad_batched(form: int, X: torch.Tensor, w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, scale_mu: float, scale_sigma: float) -> tuple:
    """K4 for `items` independent searches in one launch chain.  X: (items, N, D), w: (items, N), mu / sigma: (D,) or (items, D)."""
    if not (X.is_cuda and X.dtype == torch.float32 and X.ndim == 3):
        raise ValueError("X: expected a float32 CUDA tensor of shape (items, N, D)")
    X = as_plain_tensor(X).contiguous()
    B, n, d = X.shape
    return _grad_batched_call("evok_grad_batched", "grad", w, mu, sigma, B, n, d, lambda mu, sm, sigma, ss: (
        form, X.data_ptr(), n * d, d, w.data_ptr(), mu.data_ptr(), sm, sigma.data_ptr(), ss, B, n, d, scale_mu, scale_sigma))


def grad_batched_regen(form: int, w: torch.Tensor, mu: torch.Tensor, sigma: torch.Tensor, scale_mu: float, scale_sigma: float, *, seed: int,
                       stream_id0: int = 0) -> tuple:
    """`grad_batched` over the population that `sample_eval_batched` / `sample_batched` drew from these mu and sigma with this seed
    and stream_id0, without reading it: the rows with a non-zero weight are rebuilt from their Philox counters.  Bit-identical to
    `grad_batched` over the stored population.  w: (items, N), mu / sigma: (D,) or (items, D)."""
    if not (w.is_cuda and w.dtype == torch.float32 and w.ndim == 2):
        raise ValueError("w: expected a float32 CUDA tensor of shape (items, N)")
    B, n = w.shape
    d = mu.shape[-1]
    return _grad_batched_call("evok_grad_batched_regen", "grad_regen", w, mu, sigma, B, n, d, lambda mu, sm, sigma, ss: (
        form, w.data_ptr(), mu.data_ptr(), sm, sigma.data_ptr(), ss, B, n, d, seed, stream_id0, scale_mu, scale_sigma))


def clipup_batched_(g: torch.Tensor, velocity: torch.Tensor, center: torch.Tensor, stepsizes, momenta, max_speeds) -> None:
    """In place on contiguous (items, D) tensors: one CTA per item (per-item hyper-parameters are host scalars)."""
    B, d = center.shape
    for t, name in ((g, "g"), (velocity, "velocity"), (center, "center")):
        _rows(t, name, (B, d))
    nat.check(nat.lib().evok_clipup_batched(g.data_ptr(), B, d, velocity.data_ptr(), center.data_ptr(), _host_floats(stepsizes, B),
                                            _host_floats(momenta, B), _host_floats(max_speeds, B), nat.stream_of(g)), "evok_clipup_batched")


def sigma_update_batched_(sigma: torch.Tensor, g: torch.Tensor, lrs, exp_form: bool, lb: Optional[torch.Tensor] = None,
                          ub: Optional[torch.Tensor] = None, max_change: Optional[torch.Tensor] = None) -> None:
    """In place on contiguous (items, D) tensors; lb / ub / max_change: (items, D) tensors or None."""
    B, d = sigma.shape
    for t, name in ((sigma, "sigma"), (g, "g"), (lb, "lb"), (ub, "ub"), (max_change, "max_change")):
        if t is not None:
            _rows(t, name, (B, d))
    nat.check(nat.lib().evok_sigma_update_batched(sigma.data_ptr(), g.data_ptr(), B, d, _host_floats(lrs, B), int(bool(exp_form)), nat.ptr(lb),
                                                  nat.ptr(ub), nat.ptr(max_change), nat.stream_of(sigma)), "evok_sigma_update_batched")


# ------------------------------------------------------------------------------------------------ K8
ACT_IDS = {"none": 0, "identity": 0, "tanh": 1, "relu": 2, "sigmoid": 3}


def mlp_forward(params: torch.Tensor, obs: torch.Tensor, dims, acts, out: Optional[torch.Tensor] = None, *,
                obs_sum: Optional[torch.Tensor] = None, obs_sumsq: Optional[torch.Tensor] = None, obs_count: Optional[torch.Tensor] = None,
                min_variance: float = 1e-2, clip: Optional[tuple] = None, active: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Batched policy forward: row i of `params` (flat Linear-layer parameters) applied to row i of `obs`.
    With `obs_sum / obs_sumsq / obs_count` (the RunningNorm sums, all on the device) the observations are normalised and
    clipped while they are loaded; with `active` (bool / uint8, N) inactive policies are skipped and get zero actions."""
    _mat(params, "parameters"); _mat(obs, "observations")
    n = params.shape[0]
    dims = [int(d) for d in dims]
    act_ids = [ACT_IDS[a] if isinstance(a, str) else int(a) for a in acts]
    if obs.shape != (n, dims[0]):
        raise ValueError(f"observations: expected shape {(n, dims[0])}, got {tuple(obs.shape)}")
    if out is None:
        out = torch.empty(n, dims[-1], dtype=torch.float32, device=params.device)
    _mat(out, "out")
    d_arr = (ctypes.c_int32 * len(dims))(*dims)
    a_arr = (ctypes.c_int32 * len(act_ids))(*act_ids)
    need = nat.lib().evok_mlp_parameter_length(len(act_ids), d_arr)
    if params.shape[1] != need:
        raise ValueError(f"parameters: expected {need} columns for layer widths {dims}, got {params.shape[1]}")
    if obs_sum is None and active is None:
        with _timed("mlp_forward"):
            rc = nat.lib().evok_mlp_forward(params.data_ptr(), params.stride(0), obs.data_ptr(), obs.stride(0), out.data_ptr(), out.stride(0), n,
                                            len(act_ids), d_arr, a_arr, nat.stream_of(params))
        nat.check(rc, "evok_mlp_forward")
        return out
    if obs_sum is not None:
        _vec(obs_sum, "obs_sum", dims[0]); _vec(obs_sumsq, "obs_sumsq", dims[0])
        if obs_count is None or obs_count.dtype != torch.int64 or obs_count.numel() != 1 or not obs_count.is_cuda:
            raise ValueError("obs_count: expected a 1-element int64 CUDA tensor")
    if active is not None:
        if active.dtype == torch.bool:
            active = active.view(torch.uint8)
        if active.dtype != torch.uint8 or active.numel() != n or not active.is_cuda or not active.is_contiguous():
            raise ValueError(f"active: expected {n} contiguous bool / uint8 flags on the GPU")
    ws = None if active is None else nat.workspace(params.device, 256, "mlp")
    lo, hi = (NAN, NAN) if clip is None else (NAN if clip[0] is None else float(clip[0]), NAN if clip[1] is None else float(clip[1]))
    with _timed("mlp_forward"):
        rc = nat.lib().evok_mlp_forward_prep(params.data_ptr(), params.stride(0), obs.data_ptr(), obs.stride(0), out.data_ptr(), out.stride(0), n,
                                             len(act_ids), d_arr, a_arr, nat.ptr(obs_sum), nat.ptr(obs_sumsq), nat.ptr(obs_count),
                                             float(min_variance), lo, hi, nat.ptr(active), nat.ptr(ws), 0 if ws is None else ws.numel(),
                                             nat.stream_of(params))
    nat.check(rc, "evok_mlp_forward_prep")
    return out


def mlp_forward_shared_supported(dims) -> bool:
    """Whether `mlp_forward_shared` takes a net with these layer widths (the library's own rule: 2 to 8 layers, hidden and output
    widths <= 512, and every layer after the first small enough for its kernel to stage in shared memory)."""
    dims = [int(d) for d in dims]
    return bool(nat.lib().evok_mlp_forward_shared_supported(len(dims) - 1, (ctypes.c_int32 * len(dims))(*dims)))


def mlp_forward_shared(params: torch.Tensor, x: torch.Tensor, dims, acts) -> torch.Tensor:
    """Row i of `params` (N x L flat feed-forward parameters) applied to the SHARED input batch `x` (B x in) -> N x B x out.
    First layer: one tensor-core product of the stacked weight rows of all N networks with the batch (weights read from HBM once,
    3xTF32 = fp32 accuracy); remaining layers: per-network fp32 kernel.  Nets outside `mlp_forward_shared_supported` raise."""
    _mat(params, "parameters"); _mat(x, "x")
    dims = [int(d) for d in dims]
    act_ids = [ACT_IDS[a] if isinstance(a, str) else int(a) for a in acts]
    n, B = params.shape[0], x.shape[0]
    if x.shape[1] != dims[0]:
        raise ValueError(f"x: expected {dims[0]} columns, got {x.shape[1]}")
    if len(act_ids) != len(dims) - 1 or not mlp_forward_shared_supported(dims):
        raise ValueError(f"mlp_forward_shared does not handle layer widths {dims}: it takes 2 to 8 layers, widths <= 512 after the "
                         "input, and layers after the first that fit its shared-memory staging (use Policy.forward_shared, which "
                         "falls back to vmap)")
    d_arr = (ctypes.c_int32 * len(dims))(*dims)
    a_arr = (ctypes.c_int32 * len(act_ids))(*act_ids)
    lib = nat.lib()
    if params.shape[1] != lib.evok_mlp_parameter_length(len(act_ids), d_arr):
        raise ValueError("parameters: wrong number of columns for these layer widths")
    if x.data_ptr() % 16 != 0 or x.stride(0) % 4 != 0:  # the batch is the TMA operand: 16-byte aligned rows
        padded = torch.zeros(B, (dims[0] + 3) // 4 * 4, dtype=torch.float32, device=x.device)
        padded[:, :dims[0]] = x
        x = padded[:, :dims[0]]
    out = torch.empty(n, B, dims[-1], dtype=torch.float32, device=params.device)
    ws = nat.workspace(params.device, lib.evok_mlp_forward_shared_workspace_bytes(n, B, len(act_ids), d_arr) + 512, "mlp_shared")
    with _timed("mlp_forward_shared"):
        rc = lib.evok_mlp_forward_shared(params.data_ptr(), params.stride(0), n, x.data_ptr(), x.stride(0), B, len(act_ids), d_arr, a_arr,
                                         out.data_ptr(), ws.data_ptr(), ws.numel(), nat.stream_of(params))
    nat.check(rc, "evok_mlp_forward_shared")
    return out


# ------------------------------------------------------------------------------------------------ K6 / K7
def gemm_nt(A: torch.Tensor, B: torch.Tensor, out: Optional[torch.Tensor] = None, *, out2: Optional[torch.Tensor] = None,
            alpha: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """C = A @ B.T on the tensor cores with fp32 accuracy (3xTF32); optionally also out2 = alpha * C + bias (broadcast over rows)."""
    _mat(A, "A"); _mat(B, "B")
    M, K = A.shape
    N, K2 = B.shape
    if K != K2:
        raise ValueError(f"inner dimensions differ: {K} vs {K2}")
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=A.device)
    _mat(out, "out")
    if out2 is not None:
        _mat(out2, "out2")
    if bias is not None:
        _vec(bias, "bias", N)
    nbytes = nat.lib().evok_gemm_workspace_bytes(M, N, K)
    ws = nat.workspace(A.device, nbytes, "gemm")
    with _timed("gemm"):
        rc = nat.lib().evok_gemm_nt(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), M, N, K, out.data_ptr(), out.stride(0), nat.ptr(out2),
                                    0 if out2 is None else out2.stride(0), nat.ptr(alpha), nat.ptr(bias), ws.data_ptr(), ws.numel(),
                                    nat.stream_of(A))
    nat.check(rc, "evok_gemm_nt")
    return out


def weighted_syrk_update(Y: torch.Tensor, w: torch.Tensor, k: torch.Tensor, C: torch.Tensor, u: Optional[torch.Tensor] = None,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = k[0] * (Y^T diag(w) Y) + k[1] * C + k[2] * u u^T  -- the rank-mu + rank-1 covariance update of CMA-ES (cmaes.py:519-553)
    as one transposing pass over Y and one tensor-core GEMM whose epilogue (or split-K reduction) applies the update.
    `k`: 3 device floats.  `out` may be `C` (in place)."""
    _mat(Y, "Y"); _mat(C, "C")
    n, d = Y.shape
    _vec(w, "w", n); _vec(k, "k", 3)
    if C.shape != (d, d):
        raise ValueError(f"C: expected shape {(d, d)}, got {tuple(C.shape)}")
    if u is not None:
        _vec(u, "u", d)
    out = torch.empty_like(C) if out is None else _mat(out, "out")
    ldo = (n + 3) // 4 * 4
    lib = nat.lib()
    tws = nat.workspace(Y.device, 2 * d * ldo * 4 + 256, "syrk_operands")
    base = (tws.data_ptr() + 255) // 256 * 256
    a_w, a_p = base, base + d * ldo * 4
    nat.check(lib.evok_transpose_pair(Y.data_ptr(), Y.stride(0), n, d, w.data_ptr(), a_w, a_p, ldo, nat.stream_of(Y)), "evok_transpose_pair")
    ws = nat.workspace(Y.device, lib.evok_gemm_workspace_bytes(d, d, n), "gemm")
    with _timed("gemm"):
        rc = lib.evok_gemm_nt_affine(a_w, ldo, a_p, ldo, d, d, n, out.data_ptr(), out.stride(0), k.data_ptr(), C.data_ptr(), C.stride(0), nat.ptr(u),
                                     ws.data_ptr(), ws.numel(), nat.stream_of(Y))
    nat.check(rc, "evok_gemm_nt_affine")
    return out


def cholesky(A: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Lower Cholesky factor of a symmetric positive definite fp32 matrix (only the lower triangle of `A` is read); NaNs if `A` is not
    positive definite.  One persistent tile-dataflow kernel (csrc/evok_chol.cu)."""
    _mat(A, "A")
    n = A.shape[0]
    if A.shape[1] != n:
        raise ValueError(f"A: expected a square matrix, got {tuple(A.shape)}")
    out = torch.empty_like(A) if out is None else _mat(out, "out")
    if out.data_ptr() == A.data_ptr():
        raise ValueError("out must not alias A")
    lib = nat.lib()
    ws = nat.workspace(A.device, lib.evok_cholesky_workspace_bytes(n), "cholesky")
    with _timed("cholesky"):
        rc = lib.evok_cholesky(A.data_ptr(), A.stride(0), n, out.data_ptr(), out.stride(0), ws.data_ptr(), ws.numel(), nat.stream_of(A))
    nat.check(rc, "evok_cholesky")
    return out


def transpose_scale(X: torch.Tensor, w: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(w[:, None] * X).T as a new row-major matrix."""
    _mat(X, "X")
    rows, cols = X.shape
    if w is not None:
        _vec(w, "w", rows)
    out = torch.empty(cols, rows, dtype=torch.float32, device=X.device)
    nat.check(nat.lib().evok_transpose_scale(X.data_ptr(), X.stride(0), rows, cols, nat.ptr(w), out.data_ptr(), out.stride(0),
                                             nat.stream_of(X)), "evok_transpose_scale")
    return out


# ------------------------------------------------------------------------------------------------ batched K6 / K7 and CMA-ES glue
def _item_mat(t: torch.Tensor, name: str, core: tuple) -> tuple:
    """(tensor, n_items or None, item stride, row pitch) of a row-major matrix operand of a batched product: shape `core` (shared
    by every item: stride 0) or (items, *core) at any item stride."""
    if not (t.is_cuda and t.dtype == torch.float32 and t.ndim in (2, 3) and tuple(t.shape[-2:]) == tuple(core)):
        raise ValueError(f"{name}: expected a float32 CUDA tensor of shape {core} or (items, {core[0]}, {core[1]}), got {tuple(t.shape)} {t.dtype}")
    rows, cols = core
    # the stride of a dimension of size 1 is never stepped (torch leaves it arbitrary, even in a contiguous tensor of shape (n, 1))
    if not ((t.stride(-1) == 1 or cols == 1) and (t.stride(-2) >= cols or rows == 1)):
        raise ValueError(f"{name}: expected row-major rows (strides {t.stride()})")
    t = as_plain_tensor(t)
    ld = t.stride(-2) if rows > 1 else cols
    if t.ndim == 2:
        return t, None, 0, ld
    if t.shape[0] > 1 and t.stride(0) < 0:
        raise ValueError(f"{name}: negative item stride")
    return t, t.shape[0], t.stride(0) if t.shape[0] > 1 else 0, ld


def _item_vec(t: Optional[torch.Tensor], name: str, n: int, n_items: int) -> int:
    """Item stride of a contiguous per-item vector operand: (n,) shared -> 0, (items, n) -> n (n = 1 also takes shape (items,))."""
    if t is None:
        return 0
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise ValueError(f"{name}: expected a contiguous float32 CUDA tensor")
    if t.numel() == n and (t.ndim <= 1 or t.shape[0] == 1):
        return 0
    if t.numel() == n * n_items and t.shape[0] == n_items:
        return n
    raise ValueError(f"{name}: expected {n} values shared by the items or {n_items} x {n}, got shape {tuple(t.shape)}")


def _batch_count(*counts) -> int:
    given = {c for c in counts if c is not None}
    if len(given) > 1:
        raise ValueError(f"operands disagree on the number of items: {sorted(given)}")
    return given.pop() if given else 1


def gemm_nt_batched(A: torch.Tensor, B: torch.Tensor, out: Optional[torch.Tensor] = None, *, out2: Optional[torch.Tensor] = None,
                    alpha: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[b] = A[b] @ B[b].T for every item in one launch per 65535 items (`gemm_nt`'s 3xTF32 kernel, item = grid z; per item the
    bits of `gemm_nt` wherever its plan has one K split); optionally out2[b] = alpha[b] * out[b] + bias[b] (broadcast over rows).
    A: (M, K) or (items, M, K), B: (N, K) or (items, N, K) -- a 2-D operand is shared by every item; alpha: 1 or (items,) values,
    bias: (N,) or (items, N)."""
    A, na, sa, lda = _item_mat(A, "A", tuple(A.shape[-2:]))
    B, nb, sb, ldb = _item_mat(B, "B", tuple(B.shape[-2:]))
    M, K = A.shape[-2:]
    N, K2 = B.shape[-2:]
    if K != K2:
        raise ValueError(f"inner dimensions differ: {K} vs {K2}")
    n_items = _batch_count(na, nb, None if out is None or out.ndim < 3 else out.shape[0], None if out2 is None or out2.ndim < 3 else out2.shape[0])
    if out is None:
        out = torch.empty(n_items, M, N, dtype=torch.float32, device=A.device)
    out, _, sc, ldc = _item_mat(out, "out", (M, N))
    sc2, ldc2 = 0, 0
    if out2 is not None:
        out2, _, sc2, ldc2 = _item_mat(out2, "out2", (M, N))
    s_alpha = _item_vec(alpha, "alpha", 1, n_items)
    s_bias = _item_vec(bias, "bias", N, n_items)
    lib = nat.lib()
    ws = nat.workspace(A.device, lib.evok_gemm_nt_batched_workspace_bytes(A.data_ptr(), lda, sa, B.data_ptr(), ldb, sb, n_items, M, N, K), "gemm_batched")
    with _timed("gemm"):
        rc = lib.evok_gemm_nt_batched(A.data_ptr(), lda, sa, B.data_ptr(), ldb, sb, n_items, M, N, K, out.data_ptr(), ldc, sc, nat.ptr(out2), ldc2, sc2,
                                      nat.ptr(alpha), s_alpha, nat.ptr(bias), s_bias, ws.data_ptr(), ws.numel(), nat.stream_of(A))
    nat.check(rc, "evok_gemm_nt_batched")
    return out


def gemm_nt_affine_batched(A: torch.Tensor, B: torch.Tensor, k: torch.Tensor, out: torch.Tensor, *, E: Optional[torch.Tensor] = None,
                           u: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[b] = k[b, 0] * A[b] @ B[b].T + k[b, 1] * E[b] + k[b, 2] * outer(u[b], u[b]) for every item (`E` may be `out`).
    A / B as in `gemm_nt_batched`; k: (3,) or (items, 3); E: (M, N) or (items, M, N); u: (M,) or (items, M), needs M == N."""
    A, na, sa, lda = _item_mat(A, "A", tuple(A.shape[-2:]))
    B, nb, sb, ldb = _item_mat(B, "B", tuple(B.shape[-2:]))
    M, K = A.shape[-2:]
    N = B.shape[-2]
    if B.shape[-1] != K:
        raise ValueError(f"inner dimensions differ: {K} vs {B.shape[-1]}")
    n_items = _batch_count(na, nb, out.shape[0] if out.ndim == 3 else None)
    out, _, sc, ldc = _item_mat(out, "out", (M, N))
    se, lde = 0, 0
    if E is not None:
        E, ne, se, lde = _item_mat(E, "E", (M, N))
        _batch_count(n_items, ne)
    sk = _item_vec(k, "k", 3, n_items)
    su = _item_vec(u, "u", M, n_items)
    lib = nat.lib()
    ws = nat.workspace(A.device, lib.evok_gemm_nt_batched_workspace_bytes(A.data_ptr(), lda, sa, B.data_ptr(), ldb, sb, n_items, M, N, K), "gemm_batched")
    with _timed("gemm"):
        rc = lib.evok_gemm_nt_affine_batched(A.data_ptr(), lda, sa, B.data_ptr(), ldb, sb, n_items, M, N, K, out.data_ptr(), ldc, sc, k.data_ptr(), sk,
                                             nat.ptr(E), lde, se, nat.ptr(u), su, ws.data_ptr(), ws.numel(), nat.stream_of(A))
    nat.check(rc, "evok_gemm_nt_affine_batched")
    return out


def weighted_syrk_update_batched(Y: torch.Tensor, w: torch.Tensor, k: torch.Tensor, C: torch.Tensor, u: Optional[torch.Tensor] = None,
                                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`weighted_syrk_update` for every item: out[b] = k[b, 0] Y[b]^T diag(w[b]) Y[b] + k[b, 1] C[b] + k[b, 2] u[b] u[b]^T, as one
    transposing pass over all Y[b] and one batched GEMM whose epilogue applies the update.  Y: (items, n, d), w: (items, n),
    k: (items, 3), C: (items, d, d), u: (items, d).  `out` may be `C` (in place)."""
    if not (Y.is_cuda and Y.dtype == torch.float32 and Y.ndim == 3):
        raise ValueError("Y: expected a float32 CUDA tensor of shape (items, n, d)")
    Y = as_plain_tensor(Y).contiguous()
    B, n, d = Y.shape
    w = _rows(w, "w", (B, n))
    k = _rows(k, "k", (B, 3))
    C, nc, _, _ = _item_mat(C, "C", (d, d))
    _batch_count(B, nc)
    if u is not None:
        u = _rows(u, "u", (B, d))
    out = torch.empty(B, d, d, dtype=torch.float32, device=Y.device) if out is None else out
    ldo = (n + 3) // 4 * 4
    lib = nat.lib()
    a_w, a_p = torch.empty(2, B, d, ldo, dtype=torch.float32, device=Y.device)  # K-major operands, 16-byte aligned rows
    nat.check(lib.evok_transpose_pair_batched(Y.data_ptr(), d, n * d, n, d, w.data_ptr(), n, a_w.data_ptr(), a_p.data_ptr(), ldo, d * ldo, B,
                                              nat.stream_of(Y)), "evok_transpose_pair_batched")
    return gemm_nt_affine_batched(a_w[:, :, :n], a_p[:, :, :n], k, out, E=C, u=u)


def _tiers(tier: torch.Tensor, B: int, table: Optional[torch.Tensor] = None, name: str = "", dtype=None) -> int:
    """Checks the per-item tier indices of a padded-population stage, int32 (items,), and a device table indexed by tier (its
    first dimension, the number of tiers, is returned)."""
    if not (tier.is_cuda and tier.dtype == torch.int32 and tier.is_contiguous() and tuple(tier.shape) == (B,)):
        raise ValueError(f"tier: expected a contiguous int32 CUDA tensor of shape ({B},)")
    if table is None:
        return 0
    if not (table.is_cuda and table.dtype == dtype and table.is_contiguous() and table.ndim >= 1 and table.device == tier.device):
        raise ValueError(f"{name}: expected a contiguous {dtype} CUDA tensor indexed by tier, got {tuple(table.shape)} {table.dtype}")
    return table.shape[0]


def rank_table_batched(keys: torch.Tensor, descending: bool, table: torch.Tensor, out: Optional[torch.Tensor] = None, *,
                       tier: Optional[torch.Tensor] = None, counts: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`rank_table` for every row of keys (items, N) with one shared table (N,).  With `tier` (int32 (items,)), the padded form:
    `table` is (K, N), `counts` int32 (K,) with 1 <= counts[k] <= N, and item b ranks its first counts[tier[b]] keys with table
    row tier[b] and gets 0 on the rest (its pad rows); counting rank only, N <= 8192."""
    if not (keys.is_cuda and keys.dtype == torch.float32 and keys.ndim == 2):
        raise ValueError("keys: expected a float32 CUDA tensor of shape (items, N)")
    keys = as_plain_tensor(keys).contiguous()
    B, n = keys.shape
    out = torch.empty_like(keys) if out is None else _rows(out, "out", (B, n))
    if tier is None:
        _vec(table, "table", n)
        _rank_call("evok_rank_table_batched", keys, keys.data_ptr(), n, B, int(bool(descending)), table.data_ptr(), out.data_ptr())
        return out
    K = _tiers(tier, B, counts, "counts", torch.int32)
    if not (table.is_cuda and table.dtype == torch.float32 and table.is_contiguous() and tuple(table.shape) == (K, n)):
        raise ValueError(f"table: expected a contiguous float32 CUDA tensor of shape {(K, n)}")
    with _timed("rank"):
        rc = nat.lib().evok_rank_table_batched_tiered(keys.data_ptr(), n, B, int(bool(descending)), table.data_ptr(), tier.data_ptr(), counts.data_ptr(),
                                                      out.data_ptr(), nat.stream_of(keys))
    nat.check(rc, "evok_rank_table_batched_tiered")
    return out


def cmaes_row_weights_batched(assigned: torch.Tensor, Z: torch.Tensor, active: bool, w_pos: torch.Tensor, w_act: torch.Tensor, *,
                              tier: Optional[torch.Tensor] = None, counts: Optional[torch.Tensor] = None) -> None:
    """`cmaes_row_weights` for every item: assigned, w_pos, w_act (items, N); Z (items, N, D) with row-major rows.  With `tier`
    (int32 (items,)) and `counts` (int32 (K,)), item b uses its first counts[tier[b]] rows and gets 0 weights on the rest."""
    Z, nz, sz, ldz = _item_mat(Z, "Z", tuple(Z.shape[-2:]))
    if nz is None:
        raise ValueError("Z: expected shape (items, N, D)")
    B, n, d = Z.shape
    for t, name in ((assigned, "assigned"), (w_pos, "w_pos"), (w_act, "w_act")):
        _rows(t, name, (B, n))
    head = (assigned.data_ptr(), Z.data_ptr(), sz, ldz, B, n, d, int(bool(active)))
    if tier is None:
        nat.check(nat.lib().evok_cmaes_row_weights_batched(*head, w_pos.data_ptr(), w_act.data_ptr(), nat.stream_of(Z)), "evok_cmaes_row_weights_batched")
        return
    _tiers(tier, B, counts, "counts", torch.int32)
    nat.check(nat.lib().evok_cmaes_row_weights_batched_tiered(*head, tier.data_ptr(), counts.data_ptr(), w_pos.data_ptr(), w_act.data_ptr(),
                                                              nat.stream_of(Z)), "evok_cmaes_row_weights_batched_tiered")


def sepcma_moments_batched(X: Optional[torch.Tensor], m: torch.Tensor, s: torch.Tensor, aw: torch.Tensor, active: bool, *, seed: int = 0,
                           stream_id0: int = 0) -> tuple:
    """Separable CMA-ES moments of every item over the steps recovered from its rows, z = (x - m) / s (correctly rounded):
    local = sum_i a_i z_i, S2 = sum_i b_i z_i^2 (items, D) and wsum = sum_i b_i (items,), with the weights of `sepcma_moments` and
    q_i = ||z_i||^2 of that z.  X: (items, N, D), or None for the population that `sample_eval_batched` drew from these m and s with
    this seed and stream_id0, whose rows are rebuilt bit for bit instead of read.  m, s: (items, D); aw: (items, N)."""
    if not (aw.is_cuda and aw.dtype == torch.float32 and aw.ndim == 2):
        raise ValueError("aw: expected a float32 CUDA tensor of shape (items, N)")
    B, n = aw.shape
    d = m.shape[-1]
    aw = _rows(aw, "aw", (B, n))
    m, s = _rows(m, "m", (B, d)), _rows(s, "s", (B, d))
    if X is not None:
        if not (X.is_cuda and X.dtype == torch.float32 and X.is_contiguous() and tuple(X.shape) == (B, n, d)):
            raise ValueError(f"X: expected a contiguous float32 CUDA tensor of shape {(B, n, d)}")
        X = as_plain_tensor(X)
    local, S2 = torch.empty(B, d, dtype=torch.float32, device=aw.device), torch.empty(B, d, dtype=torch.float32, device=aw.device)
    wsum = torch.empty(B, dtype=torch.float32, device=aw.device)
    lib = nat.lib()
    ws = nat.workspace(aw.device, lib.evok_sepcma_moments_batched_workspace_bytes(B, n, d), "grad_batched")
    with _timed("sepcma_moments"):
        rc = lib.evok_sepcma_moments_batched(nat.ptr(X), n * d, d, m.data_ptr(), s.data_ptr(), aw.data_ptr(), int(bool(active)), B, n, d, seed,
                                             stream_id0, local.data_ptr(), S2.data_ptr(), wsum.data_ptr(), ws.data_ptr(), ws.numel(),
                                             nat.stream_of(aw))
    nat.check(rc, "evok_sepcma_moments_batched")
    return local, S2, wsum


def _item_steps(steps, B: int) -> Optional[torch.Tensor]:
    """None for a shared host counter (an int), else `steps` checked as one int64 CUDA counter per item, (items,) contiguous."""
    if not isinstance(steps, torch.Tensor):
        return None
    if not (steps.is_cuda and steps.dtype == torch.int64 and steps.is_contiguous() and tuple(steps.shape) == (B,)):
        raise ValueError(f"steps: expected an int or a contiguous int64 CUDA tensor of shape ({B},), got {tuple(steps.shape)} {steps.dtype}")
    return steps


def sepcma_update_batched(local: torch.Tensor, S2: torch.Tensor, wsum: torch.Tensor, m: torch.Tensor, p_sigma: torch.Tensor, p_c: torch.Tensor,
                          sigma: torch.Tensor, C: torch.Tensor, A: torch.Tensor, s: torch.Tensor, consts, csa_squared: bool, *, steps,
                          decompose_C_freq, stdev_min: Optional[float] = None, stdev_max: Optional[float] = None,
                          tier: Optional[torch.Tensor] = None) -> None:
    """`sepcma_update` for every item, one CTA each, in place: m, p_sigma, p_c, C, A, s, local, S2 (items, D), sigma, wsum (items,).
    The 10 constants, `decompose_C_freq` and the stdev bounds are shared.  `steps`: the generation counter, an int shared by every
    item, or an int64 CUDA tensor (items,) of per-item counters that drive each item's h_sig and decomposition schedule and are
    incremented in place.  With `tier` (int32 (items,), per-item counters), `consts` is a float32 CUDA table (K, 10) and
    `decompose_C_freq` an int64 CUDA table (K,), both read at row tier[b] for item b."""
    B, d = m.shape
    for t, name in ((local, "local"), (S2, "S2"), (m, "m"), (p_sigma, "p_sigma"), (p_c, "p_c"), (C, "C"), (A, "A"), (s, "s")):
        _rows(t, name, (B, d))
    for t, name in ((sigma, "sigma"), (wsum, "wsum")):
        _rows(t, name, (B,))
    lo = NAN if stdev_min is None else float(stdev_min)
    hi = NAN if stdev_max is None else float(stdev_max)
    if tier is not None:
        steps_dev = _item_steps(steps, B)
        if steps_dev is None:
            raise ValueError("steps: the tiered update takes per-item counters")
        K = _tiers(tier, B, consts, "consts", torch.float32)
        if tuple(consts.shape) != (K, 10) or _tiers(tier, B, decompose_C_freq, "decompose_C_freq", torch.int64) != K or decompose_C_freq.ndim != 1:
            raise ValueError(f"consts, decompose_C_freq: expected tables of shapes ({K}, 10) and ({K},)")
        with _timed("sepcma_update"):
            rc = nat.lib().evok_sepcma_update_batched_tiered(local.data_ptr(), S2.data_ptr(), wsum.data_ptr(), B, d, m.data_ptr(), p_sigma.data_ptr(),
                                                             p_c.data_ptr(), sigma.data_ptr(), C.data_ptr(), A.data_ptr(), s.data_ptr(), steps_dev.data_ptr(),
                                                             tier.data_ptr(), consts.data_ptr(), decompose_C_freq.data_ptr(), int(bool(csa_squared)), lo, hi,
                                                             nat.stream_of(m))
        nat.check(rc, "evok_sepcma_update_batched_tiered")
        return
    if int(decompose_C_freq) < 1:
        raise ValueError("decompose_C_freq: expected a positive integer")
    steps_dev = _item_steps(steps, B)
    lib = nat.lib()
    head = (local.data_ptr(), S2.data_ptr(), wsum.data_ptr(), B, d, m.data_ptr(), p_sigma.data_ptr(), p_c.data_ptr(), sigma.data_ptr(), C.data_ptr(),
            A.data_ptr(), s.data_ptr())
    tail = (_host_floats(consts, 10), int(bool(csa_squared)), int(decompose_C_freq), lo, hi, nat.stream_of(m))
    with _timed("sepcma_update"):
        if steps_dev is None:
            rc, entry = lib.evok_sepcma_update_batched(*head, int(steps), *tail), "evok_sepcma_update_batched"
        else:
            rc, entry = lib.evok_sepcma_update_batched_steps(*head, steps_dev.data_ptr(), *tail), "evok_sepcma_update_batched_steps"
    nat.check(rc, entry)


def cmaes_vector_update_batched(local_disp: torch.Tensor, shaped_disp: torch.Tensor, m: torch.Tensor, p_sigma: torch.Tensor, p_c: torch.Tensor,
                                sigma: torch.Tensor, consts, csa_squared: bool, k_out: torch.Tensor, *, steps,
                                tier: Optional[torch.Tensor] = None) -> None:
    """`cmaes_vector_update` for every item, one CTA each, in place: m, p_sigma, p_c, local / shaped (items, D), sigma (items,),
    k_out (items, 3).  The 10 constants are shared.  `steps`: the generation counter, an int shared by every item, or an int64
    CUDA tensor (items,) of per-item counters that drive each item's h_sig and are incremented in place.  With `tier` (int32
    (items,), per-item counters), `consts` is a float32 CUDA table (K, 10) read at row tier[b] for item b."""
    B, d = m.shape
    for t, name in ((local_disp, "local_disp"), (shaped_disp, "shaped_disp"), (m, "m"), (p_sigma, "p_sigma"), (p_c, "p_c")):
        _rows(t, name, (B, d))
    _rows(sigma.view(B, 1) if sigma.numel() == B and sigma.is_contiguous() else sigma, "sigma", (B, 1))
    _rows(k_out, "k_out", (B, 3))
    steps_dev = _item_steps(steps, B)
    lib = nat.lib()
    head = (local_disp.data_ptr(), shaped_disp.data_ptr(), B, d, m.data_ptr(), p_sigma.data_ptr(), p_c.data_ptr(), sigma.data_ptr())
    if tier is not None:
        if steps_dev is None:
            raise ValueError("steps: the tiered update takes per-item counters")
        K = _tiers(tier, B, consts, "consts", torch.float32)
        if tuple(consts.shape) != (K, 10):
            raise ValueError(f"consts: expected a table of shape ({K}, 10)")
        nat.check(lib.evok_cmaes_vector_update_batched_tiered(*head, steps_dev.data_ptr(), tier.data_ptr(), consts.data_ptr(), int(bool(csa_squared)),
                                                              k_out.data_ptr(), nat.stream_of(m)), "evok_cmaes_vector_update_batched_tiered")
        return
    tail = (_host_floats(consts, 10), int(bool(csa_squared)), k_out.data_ptr(), nat.stream_of(m))
    if steps_dev is None:
        nat.check(lib.evok_cmaes_vector_update_batched(*head, int(steps), *tail), "evok_cmaes_vector_update_batched")
    else:
        nat.check(lib.evok_cmaes_vector_update_batched_steps(*head, steps_dev.data_ptr(), *tail), "evok_cmaes_vector_update_batched_steps")


LMMAES_MAX_VECTORS, LMMAES_MAX_POPSIZE = 64, 128  # EVOK_LMMAES_MAX_VECTORS, EVOK_LMMAES_MAX_POPSIZE


def _lmmaes_operands(y: torch.Tensor, sigma: torch.Tensor, M: torch.Tensor, G: torch.Tensor, k: int, consts) -> tuple:
    """Checks the state operands of the LM-MA-ES stages: y (items, D), sigma (items,), M (items, m, D), G (items, m, m), the
    2 + 2m float64 constants (c_sigma, mu_eff, c_d[m], c_c[m]); returns (items, D, m, the constants as a C double array)."""
    if not (y.is_cuda and y.dtype == torch.float32 and y.ndim == 2):
        raise ValueError("y: expected a float32 CUDA tensor of shape (items, D)")
    B, d = y.shape
    if not (M.is_cuda and M.dtype == torch.float32 and M.ndim == 3 and M.shape[0] == B and M.shape[2] == d):
        raise ValueError(f"M: expected a float32 CUDA tensor of shape ({B}, m, {d})")
    m = M.shape[1]
    _rows(y, "y", (B, d))
    _rows(sigma, "sigma", (B,))
    _rows(M, "M", (B, m, d))
    _rows(G, "G", (B, m, m))
    for t, name in ((sigma, "sigma"), (M, "M"), (G, "G")):
        if t.device != y.device:
            raise ValueError(f"{name}: expected on {y.device}, got {t.device}")
    if len(consts) != 2 + 2 * m:
        raise ValueError(f"consts: expected {2 + 2 * m} values (c_sigma, mu_eff, c_d[m], c_c[m]), got {len(consts)}")
    return B, d, m, (ctypes.c_double * len(consts))(*[float(c) for c in consts])


def _lmmaes_ws(device: torch.device, B: int, n: int, d: int, m: int) -> torch.Tensor:
    return nat.workspace(device, nat.lib().evok_lmmaes_workspace_bytes(B, n, d, m), "lmmaes")


def lmmaes_ask_batched(y: torch.Tensor, sigma: torch.Tensor, M: torch.Tensor, G: torch.Tensor, k: int, consts, popsize: int, *, seed: int,
                       stream_id0: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The LM-MA-ES ask of every item, (items, popsize, D): x_i = y + sigma d_i with d_i the step of z_i through the first k vectors
    of M, z_i of item b the row of `sample_batched` with this seed on stream stream_id0 + b.  Three launches per item chunk (one
    with k = 0, then x = fmaf(sigma, z, y))."""
    B, d, m, c = _lmmaes_operands(y, sigma, M, G, k, consts)
    out = torch.empty(B, popsize, d, dtype=torch.float32, device=y.device) if out is None else _rows(out, "out", (B, popsize, d))
    ws = _lmmaes_ws(y.device, B, popsize, d, m)
    with _timed("lmmaes_ask"):
        rc = nat.lib().evok_lmmaes_ask_batched(out.data_ptr(), y.data_ptr(), sigma.data_ptr(), M.data_ptr(), G.data_ptr(), B, popsize, d, m, int(k),
                                               c, seed, stream_id0, ws.data_ptr(), ws.numel(), nat.stream_of(y))
    nat.check(rc, "evok_lmmaes_ask_batched")
    return out


def lmmaes_tell_batched(X: torch.Tensor, aw: torch.Tensor, y: torch.Tensor, sigma: torch.Tensor, p_sigma: torch.Tensor, M: torch.Tensor,
                        G: torch.Tensor, k: int, consts) -> tuple:
    """The LM-MA-ES tell of every item from its rows X (items, popsize, D) and their rank weights aw (items, popsize): the new
    (y, sigma, p_sigma, M, G), all new tensors.  Four launches per item chunk."""
    B, d, m, c = _lmmaes_operands(y, sigma, M, G, k, consts)
    if not (aw.is_cuda and aw.dtype == torch.float32 and aw.ndim == 2 and aw.shape[0] == B):
        raise ValueError(f"aw: expected a float32 CUDA tensor of shape ({B}, popsize)")
    n = aw.shape[1]
    _rows(aw, "aw", (B, n))
    _rows(X, "X", (B, n, d))
    _rows(p_sigma, "p_sigma", (B, d))
    outs = (torch.empty_like(y), torch.empty_like(sigma), torch.empty_like(p_sigma), torch.empty_like(M), torch.empty_like(G))
    ws = _lmmaes_ws(y.device, B, n, d, m)
    with _timed("lmmaes_tell"):
        rc = nat.lib().evok_lmmaes_tell_batched(X.data_ptr(), aw.data_ptr(), y.data_ptr(), sigma.data_ptr(), p_sigma.data_ptr(), M.data_ptr(),
                                                G.data_ptr(), B, n, d, m, int(k), c, *(t.data_ptr() for t in outs), ws.data_ptr(), ws.numel(),
                                                nat.stream_of(y))
    nat.check(rc, "evok_lmmaes_tell_batched")
    return outs


XNES_MAX_D = 96  # EVOK_XNES_MAX_D


def sym_expm_pair_batched(S: torch.Tensor) -> tuple:
    """(expm(S) - I, expm(-S) - I) of every symmetric matrix of S (items, D, D), 1 <= D <= XNES_MAX_D, one CTA per item: the
    expm1 form, which keeps the relative precision of a tiny S.  Both are new tensors."""
    if not (S.is_cuda and S.dtype == torch.float32 and S.ndim == 3 and S.shape[1] == S.shape[2]):
        raise ValueError(f"S: expected a float32 CUDA tensor of shape (items, D, D), got {tuple(S.shape)} {S.dtype}")
    B, d, _ = S.shape
    S = _rows(S.contiguous(), "S", (B, d, d))
    Fp, Fm = torch.empty_like(S), torch.empty_like(S)
    with _timed("sym_expm_pair"):
        rc = nat.lib().evok_sym_expm_pair_batched(S.data_ptr(), B, d, Fp.data_ptr(), Fm.data_ptr(), nat.stream_of(S))
    nat.check(rc, "evok_sym_expm_pair_batched")
    return Fp, Fm


def xnes_tell_batched(X: torch.Tensor, w: torch.Tensor, mu: torch.Tensor, A: torch.Tensor, A_inv: torch.Tensor, lr_mu: float, lr_A: float) -> tuple:
    """The XNES update of every item from its rows X (items, N, D) and their utilities w (items, N), centred where the ranking
    needs it: z = A_inv (x - mu) for the rows with a non-zero weight, d = sum w z, S = (lr_A / 2)(sum w z z^T - (sum w) I), and
    the new (mu + A (lr_mu d), A + A (e^S - I), A_inv + (e^-S - I) A_inv), all new tensors.  One launch per 65535 items."""
    if not (mu.is_cuda and mu.dtype == torch.float32 and mu.ndim == 2):
        raise ValueError("mu: expected a float32 CUDA tensor of shape (items, D)")
    B, d = mu.shape
    if not (w.is_cuda and w.dtype == torch.float32 and w.ndim == 2 and w.shape[0] == B):
        raise ValueError(f"w: expected a float32 CUDA tensor of shape ({B}, N)")
    n = w.shape[1]
    w, mu = _rows(w, "w", (B, n)), _rows(mu, "mu", (B, d))
    X, A, A_inv = _rows(X, "X", (B, n, d)), _rows(A, "A", (B, d, d)), _rows(A_inv, "A_inv", (B, d, d))
    outs = (torch.empty_like(mu), torch.empty_like(A), torch.empty_like(A_inv))
    with _timed("xnes_tell"):
        rc = nat.lib().evok_xnes_tell_batched(X.data_ptr(), w.data_ptr(), mu.data_ptr(), A.data_ptr(), A_inv.data_ptr(), B, n, d, float(lr_mu),
                                              float(lr_A), *(t.data_ptr() for t in outs), nat.stream_of(mu))
    nat.check(rc, "evok_xnes_tell_batched")
    return outs


RESTART_CRITERIA = ("tol_fun", "tol_x", "tol_x_up", "max_condition", "min_fitness_stdev", "max_generations")  # bits 0-5; bit 6: non-finite
# bit 7 (BIPOP only): a small run has used half the evaluations of the item's latest large run; it has no threshold


def cma_restart_batched(separable: bool, f: torch.Tensor, X: Optional[torch.Tensor], maximize: bool, item_steps: torch.Tensor, m: torch.Tensor,
                        sigma: torch.Tensor, p_sigma: torch.Tensor, p_c: torch.Tensor, C: torch.Tensor, A: torch.Tensor, s: Optional[torch.Tensor],
                        history: torch.Tensor, best_x: torch.Tensor, best_f: torch.Tensor, num_restarts: torch.Tensor, stop_flags: torch.Tensor,
                        sigma0: torch.Tensor, lb: torch.Tensor, ub: torch.Tensor, thresholds, *, seed: int, m_draw: Optional[torch.Tensor] = None,
                        s_draw: Optional[torch.Tensor] = None, draw_seed: int = 0, tier: Optional[torch.Tensor] = None,
                        tier_counts: Optional[torch.Tensor] = None, tier_history: Optional[torch.Tensor] = None,
                        num_evaluations: Optional[torch.Tensor] = None, regime: Optional[torch.Tensor] = None,
                        large_tier: Optional[torch.Tensor] = None, large_evaluations: Optional[torch.Tensor] = None,
                        small_evaluations: Optional[torch.Tensor] = None, last_large_evaluations: Optional[torch.Tensor] = None,
                        run_stdev: Optional[torch.Tensor] = None, n_large: int = 0, popsize0: int = 0) -> None:
    """The restart stage of every item after its update, in place (include/evok.h, evok_cma_restart_batched): best ever, history,
    stop flags and the re-initialisation of the items that met a criterion.  f (items, N); X (items, N, D), or None for a separable
    population rebuilt from (draw_seed, stream b) with m_draw / s_draw (items, D); item_steps, num_restarts int64 (items,); m, p_sigma,
    p_c, best_x, lb, ub (items, D); C, A (items, D, D), separable (items, D) with s; sigma, sigma0, best_f (items,); history
    (items, H); stop_flags int32 (items,); `thresholds` the 6 criteria of RESTART_CRITERIA, None = off; `seed` the Philox key of
    the new centres.  With `tier` (int32 (items,), in place), the padded form (evok_cma_restart_batched_tiered): item b uses its
    first tier_counts[tier[b]] values and tier_history[tier[b]] history slots (tables int32 and int64 (K,)), num_evaluations
    (int64 (items,)) grows by its count, and a restarted item moves one tier up.  With `regime` as well, the BIPOP form
    (evok_cma_restart_batched_bipop): sigma0 is the default step size; regime, large_tier int32 (items,), large_evaluations,
    small_evaluations, last_large_evaluations int64 (items,) and run_stdev (items,) are the per-item policy state, in place; tiers
    0..n_large-1 of the tables are the ladder from popsize0, tier n_large + (lambda - popsize0) a small run of size lambda."""
    B, n = f.shape
    d = m.shape[-1]
    f = _rows(f, "f", (B, n))
    for t, name in ((m, "m"), (p_sigma, "p_sigma"), (p_c, "p_c"), (best_x, "best_x"), (lb, "lb"), (ub, "ub")):
        _rows(t, name, (B, d))
    for t, name in ((sigma, "sigma"), (sigma0, "sigma0"), (best_f, "best_f")):
        _rows(t, name, (B,))
    for t, name in ((C, "C"), (A, "A")):
        # the stage reads the diagonals and writes I: a matrix may be row- or column-major (torch's batched Cholesky is the latter)
        if not (t.is_cuda and t.dtype == torch.float32 and (t.is_contiguous() or (not separable and t.mT.is_contiguous()))
                and tuple(t.shape) == ((B, d) if separable else (B, d, d))):
            raise ValueError(f"{name}: expected a float32 CUDA tensor of shape {(B, d) if separable else (B, d, d)}, contiguous (or its "
                             "transposes contiguous)")
    if separable:
        _rows(s, "s", (B, d))
    if not (history.is_cuda and history.dtype == torch.float32 and history.is_contiguous() and history.ndim == 2 and history.shape[0] == B):
        raise ValueError(f"history: expected a contiguous float32 CUDA tensor of shape ({B}, H)")
    for t, name, dt in ((item_steps, "item_steps", torch.int64), (num_restarts, "num_restarts", torch.int64), (stop_flags, "stop_flags", torch.int32)):
        if not (t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == (B,)):
            raise ValueError(f"{name}: expected a contiguous {dt} CUDA tensor of shape ({B},)")
    if X is not None:
        if not (X.is_cuda and X.dtype == torch.float32 and X.is_contiguous() and tuple(X.shape) == (B, n, d)):
            raise ValueError(f"X: expected a contiguous float32 CUDA tensor of shape {(B, n, d)}")
    elif not separable or m_draw is None or s_draw is None:
        raise ValueError("X: the population is needed, except for a separable one rebuilt from m_draw and s_draw")
    else:
        m_draw, s_draw = _rows(m_draw, "m_draw", (B, d)), _rows(s_draw, "s_draw", (B, d))
    th = [NAN if t is None else float(t) for t in thresholds]
    if tier is not None:
        K = _tiers(tier, B, tier_counts, "tier_counts", torch.int32)
        if _tiers(tier, B, tier_history, "tier_history", torch.int64) != K:
            raise ValueError("tier_counts and tier_history must have one entry per tier")
        if not (num_evaluations is not None and num_evaluations.is_cuda and num_evaluations.dtype == torch.int64 and num_evaluations.is_contiguous()
                and tuple(num_evaluations.shape) == (B,)):
            raise ValueError(f"num_evaluations: expected a contiguous int64 CUDA tensor of shape ({B},)")
    if regime is not None:
        if tier is None:
            raise ValueError("the BIPOP stage is the tiered one with a policy: give `tier` and its tables with `regime`")
        for t, name, dt in ((regime, "regime", torch.int32), (large_tier, "large_tier", torch.int32), (large_evaluations, "large_evaluations", torch.int64),
                            (small_evaluations, "small_evaluations", torch.int64), (last_large_evaluations, "last_large_evaluations", torch.int64)):
            if not (t is not None and t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == (B,)):
                raise ValueError(f"{name}: expected a contiguous {dt} CUDA tensor of shape ({B},)")
        _rows(run_stdev, "run_stdev", (B,))
    with _timed("cma_restart"):
        args = (int(bool(separable)), f.data_ptr(), nat.ptr(X), n * d, d, nat.ptr(m_draw), nat.ptr(s_draw), int(draw_seed), B, n, d, int(bool(maximize)),
                item_steps.data_ptr(), m.data_ptr(), sigma.data_ptr(), p_sigma.data_ptr(), p_c.data_ptr(), C.data_ptr(), A.data_ptr(), nat.ptr(s),
                history.data_ptr(), history.shape[1], best_x.data_ptr(), best_f.data_ptr(), num_restarts.data_ptr(), stop_flags.data_ptr(),
                sigma0.data_ptr(), lb.data_ptr(), ub.data_ptr(), d, _host_floats(th, 6), int(seed))
        if regime is not None:
            rc = nat.lib().evok_cma_restart_batched_bipop(*args, tier.data_ptr(), tier_counts.data_ptr(), tier_history.data_ptr(), K,
                                                          num_evaluations.data_ptr(), regime.data_ptr(), large_tier.data_ptr(),
                                                          large_evaluations.data_ptr(), small_evaluations.data_ptr(), last_large_evaluations.data_ptr(),
                                                          run_stdev.data_ptr(), int(n_large), int(popsize0), nat.stream_of(f))
            nat.check(rc, "evok_cma_restart_batched_bipop")
            return
        if tier is not None:
            rc = nat.lib().evok_cma_restart_batched_tiered(*args, tier.data_ptr(), tier_counts.data_ptr(), tier_history.data_ptr(), K,
                                                           num_evaluations.data_ptr(), nat.stream_of(f))
            nat.check(rc, "evok_cma_restart_batched_tiered")
            return
        rc = nat.lib().evok_cma_restart_batched(*args, nat.stream_of(f))
    nat.check(rc, "evok_cma_restart_batched")
