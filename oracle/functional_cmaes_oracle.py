"""Float64 references for the batched functional CMA-ES (`algorithms/functional/funccmaes.py`), shared by its tests.

* `stable_rank_table`: the ranking of `rank_table` / `rank_table_batched` (stable, -0 == +0, NaN the largest value) on a
  (items, N) array of keys, vectorised over the items.
* `reference_generation`: one generation of `es_oracle.cmaes_update` for one item, from the state under test (its own fp32
  state and learning rates) and fed that state's own z, y and fitnesses, optionally with one of `MUTATIONS` -- the wrong
  algorithms a batched implementation can plausibly compute, which the tests must tell apart from the right one.
* `tell_bound`: per item, the largest |kernel - reference| / bound over the new state, with the first-order bound of a tell
  whose z comes from a backward-stable triangular solve (the K7 bound for the SYRK), carried through the stdev clamp.
"""

from __future__ import annotations

import numpy as np
import torch

from . import es_oracle as O

EPS = 2.0 ** -24
BK = 32
CHUNK = 4
F32 = np.float32

# the one-generation mutations of `reference_generation`; the two "neighbour_*" ones are applied by `tell_bound`, which owns the
# batch: item b is ranked with item b+1's fitnesses, or recombines item b+1's rows
MUTATIONS = ("sense_flipped", "neighbour_fitness", "neighbour_rows", "h_sig_one", "m_new_sigma", "csa_swapped", "no_active", "k2_no_wpc",
             "clamp_old_sigma")


def gamma(K: int) -> float:
    """The K6 / K7 bound factor (DESIGN, "Accuracy of K6 / K7") of a one-split product over K."""
    kbps = -(-K // BK)
    k_chunk = 2 * 3 * (BK // 8) * min(kbps, CHUNK) + -(-kbps // CHUNK)
    return 3 * 2.0 ** -20 + EPS * (k_chunk + 1 + 2)


def stable_rank_table(keys: np.ndarray, descending: bool, table: np.ndarray) -> np.ndarray:
    """out[b, i] = table[position of keys[b, i] in the stable order of row b] (position 0 = the largest key if `descending`).
    Ties keep ascending index order in both senses, -0 and +0 are equal, NaN is larger than +inf (torch's order)."""
    keys = np.asarray(keys, dtype=F32)
    keys = keys.reshape(-1, keys.shape[-1])
    if descending:
        nan = np.isnan(keys)
        neg = np.where(nan, 0.0, -keys.astype(np.float64))
        # np.lexsort is stable and sorts by its last key first: NaN rows first, then by decreasing value
        order = np.stack([np.lexsort((neg[b], ~nan[b])) for b in range(keys.shape[0])]) if keys.size else np.zeros(keys.shape, np.int64)
    else:
        order = np.argsort(keys, axis=-1, kind="stable")
    ranks = np.empty_like(order)
    np.put_along_axis(ranks, order, np.broadcast_to(np.arange(keys.shape[-1]), keys.shape), axis=-1)
    return np.asarray(table, dtype=F32)[ranks]


def flat_state(state):
    """The state with its batch dimensions flattened into one item axis (B, ...)."""
    d = state.center.shape[-1]
    return state._replace(center=state.center.reshape(-1, d), sigma=state.sigma.reshape(-1), C=state.C.reshape(-1, d, d),
                          A=state.A.reshape(-1, d, d), p_sigma=state.p_sigma.reshape(-1, d), p_c=state.p_c.reshape(-1, d))


def oracle_state(state, b: int) -> O.CMAESState:
    """Item b of a flat state as an oracle state: its fp32 tensors, and the learning rates and weights of the state under test
    (bit for bit those of CMAES; the oracle's own differ in the last bits)."""
    hp = state.hyperparameters
    d = state.center.shape[-1]
    o = O.CMAESState(d, hp.popsize, float(state.sigma[b]), state.center[b].cpu().numpy(), active=state.active, csa_squared=state.csa_squared,
                     stdev_min=state.stdev_min, stdev_max=state.stdev_max)
    o.c_m, o.c_sigma, o.damp_sigma, o.c_c, o.c_1, o.c_mu = hp.c_m, hp.c_sigma, hp.damp_sigma, hp.c_c, hp.c_1, hp.c_mu
    o.variance_discount_sigma, o.variance_discount_c, o.unbiased_expectation = hp.variance_discount_sigma, hp.variance_discount_c, hp.unbiased_expectation
    o.weights = hp.weights.cpu().numpy().astype(F32)
    o.decompose_C_freq = hp.decompose_C_freq
    for name in ("p_sigma", "p_c", "C", "A"):
        setattr(o, name, getattr(state, name)[b].cpu().numpy().astype(F32))
    o.sigma = F32(state.sigma[b].item())
    o.steps = state.generation
    return o


def reference_generation(o: O.CMAESState, Z, Y, f, sense: str, mutation=None) -> dict:
    """`es_oracle.cmaes_update` on the oracle state `o` (updated in place) up to and including the stdev clamp, without the
    decomposition, with an optional mutation.  Returns h_sig, the margin of its comparison, the assigned weights and the
    stdevs sigma' sqrt(diag C) before the clamp."""
    Z, Y = np.asarray(Z, np.float64), np.asarray(Y, np.float64)
    if mutation == "sense_flipped":
        sense = "min" if sense == "max" else "max"
    aw = O.cmaes_assign_weights(o, f, sense)
    local, shaped = O.cmaes_recombine(o, Z, Y, aw)
    sig0, m0 = o.sigma, o.m.copy()
    csa = o.csa_squared if mutation != "csa_swapped" else not o.csa_squared
    # cmaes_vector_step, with the mutations' hooks
    o.m = (m0 + F32(o.c_m) * sig0 * shaped.astype(F32)).astype(F32)
    o.p_sigma = (F32(1 - o.c_sigma) * o.p_sigma + F32(o.variance_discount_sigma) * local.astype(F32)).astype(F32)
    pnorm = float(np.sqrt(np.sum(o.p_sigma.astype(np.float64) ** 2)))
    expo = (pnorm**2 / o.d - 1) / 2 if csa else pnorm / o.unbiased_expectation - 1
    o.sigma = F32(sig0 * np.exp(F32((o.c_sigma / o.damp_sigma) * expo)))
    h, margin = O.cmaes_h_sig(o, pnorm)
    if mutation == "h_sig_one":
        h = 1.0
    o.p_c = (F32(1 - o.c_c) * o.p_c + F32(h * o.variance_discount_c) * shaped.astype(F32)).astype(F32)
    if mutation == "m_new_sigma":
        o.m = (m0 + F32(o.c_m) * o.sigma * shaped.astype(F32)).astype(F32)
    c1a, wpc = O.cmaes_covariance_coefficients(o, h)
    if mutation == "k2_no_wpc":
        wpc = 1.0  # k2 = c1a
    w = aw.astype(np.float64) if mutation == "no_active" else O.cmaes_active_weights(o, Z, aw)
    O.cmaes_covariance_update(o, Y, w, c1a, wpc)
    stdevs = float(o.sigma) * np.sqrt(np.diag(o.C).astype(np.float64))
    if mutation == "clamp_old_sigma":
        new_sigma, o.sigma = o.sigma, sig0
        O.cmaes_limit_stdev(o)
        o.sigma = new_sigma
    else:
        O.cmaes_limit_stdev(o)
    return dict(h=h, margin=margin, aw=aw, stdevs=stdevs)


def tell_bound(state, x, f, new, mutation=None, items=None, record=None) -> list:
    """Per item of `items` (default: all) of a flat state: max over m, p_sigma, p_c, sigma and C of |new - reference| / bound.
    The reference (float64 sums, fp32 state) gets the tell's own y = (x - m) / sigma and z = A^-1 y solved in float64.  The
    kernel's z comes from a backward-stable TRSM: |z^ - z| <= gamma_D |A^-1| |A| |z^|, carried to the sums, the vector update and
    the covariance update to first order, with the K7 bound for the SYRK; the stdev clamp adds |C'_ii| (2 e_sigma / sigma' + 8 eps)
    on the diagonal.  `record` (a list) receives each item's reference outcome (`reference_generation`'s dict)."""
    hp = state.hyperparameters
    B, n, d = x.shape
    dev = x.device
    items = list(range(B)) if items is None else list(items)
    idx = torch.as_tensor(items, device=dev)
    m, sig, A, C = state.center[idx], state.sigma[idx], state.A[idx], state.C[idx]
    xs, fs = x[idx], f[idx]
    y = (xs - m[:, None, :]) / sig[:, None, None]
    A64 = A.double()
    z64 = torch.linalg.solve_triangular(A64.mT, y.double(), upper=True, left=False)
    gD = d * EPS / (1 - d * EPS)
    dz = gD * (z64.abs() @ (torch.linalg.inv(A64).abs() @ A64.abs()).mT) + EPS * z64.abs()
    sense = "max" if state.maximize else "min"
    aw = torch.stack([torch.as_tensor(O.cmaes_assign_weights(oracle_state(state, b), f[b].cpu().numpy(), sense)) for b in items]).to(dev).double()
    wp = aw.clamp_min(0)
    gn = n * EPS
    e_local = (wp[:, :, None] * dz).sum(1) + gn * (wp[:, :, None] * z64.abs()).sum(1)
    shaped = (wp[:, :, None] * y.double()).sum(1)
    e_shaped = gn * (wp[:, :, None] * y.double().abs()).sum(1)
    s = sig.double()[:, None]
    e_m = hp.c_m * s * e_shaped + 4 * EPS * (m.double().abs() + hp.c_m * s * shaped.abs())
    ps_new, pc_new, sig_new, C_new = new.p_sigma[idx].double(), new.p_c[idx].double(), new.sigma[idx].double(), new.C[idx].double()
    e_ps = hp.variance_discount_sigma * e_local + 4 * EPS * ((1 - hp.c_sigma) * state.p_sigma[idx].double().abs() + ps_new.abs())
    e_pn = e_ps.norm(dim=-1)
    pn = ps_new.norm(dim=-1)
    slope = (pn / d) if state.csa_squared else torch.full_like(pn, 1 / hp.unbiased_expectation)
    e_sigma = sig_new * ((hp.c_sigma / hp.damp_sigma) * slope * e_pn + 8 * EPS)
    e_pc = hp.variance_discount_c * e_shaped + 4 * EPS * ((1 - hp.c_c) * state.p_c[idx].double().abs() + pc_new.abs())
    # active weights: w = D aw / ||z||^2 for aw <= 0, so |dw| <= |w| 2 sum|z||dz| / ||z||^2
    zn2 = (z64 * z64).sum(-1)
    w_act = torch.where(aw > 0, aw, d * aw / zn2) if state.active else aw
    e_w = torch.where(aw > 0, torch.zeros_like(aw), w_act.abs() * 2 * (z64.abs() * dz).sum(-1) / zn2) if state.active else torch.zeros_like(aw)
    Y = y.double()
    S_abs = (Y.abs().mT * w_act.abs()[:, None, :]) @ Y.abs()
    e_S = gamma(n) * S_abs + (Y.abs().mT * e_w[:, None, :]) @ Y.abs()
    pc = pc_new
    k2 = hp.c_1 * (hp.c_1 / (hp.c_1 + 1e-23))  # c1a * weighted_pc^2 <= c_1 (h = 1)
    e_C = (hp.c_mu * e_S + 2 * k2 * pc.abs()[:, :, None] * e_pc[:, None, :]
           + 8 * EPS * (hp.c_mu * S_abs + C.double().abs() + k2 * pc.abs()[:, :, None] * pc.abs()[:, None, :] + C_new.abs()))
    if state.stdev_min is not None or state.stdev_max is not None:
        diag = torch.diagonal(e_C, dim1=-2, dim2=-1)
        diag += torch.diagonal(C_new, dim1=-2, dim2=-1).abs() * (2 * e_sigma / sig_new + 8 * EPS)[:, None]
    ratios = []
    for j, b in enumerate(items):
        o = oracle_state(state, b)
        fb, Zb, Yb = f[b], z64[j], y[j]
        if mutation in ("neighbour_fitness", "neighbour_rows") and B > 1:
            nb = (b + 1) % B
            if mutation == "neighbour_fitness":
                fb = f[nb]
            else:
                yn = (x[nb] - state.center[nb]) / state.sigma[nb]
                Yb, Zb = yn, torch.linalg.solve_triangular(state.A[nb].double().mT, yn.double(), upper=True, left=False)
        out = reference_generation(o, Zb.cpu().numpy(), Yb.cpu().numpy(), fb.cpu().numpy(), sense, mutation)
        if record is not None:
            record.append(out)
        r = 0.0
        for got, ref, e in ((new.center[b], o.m, e_m[j]), (new.p_sigma[b], o.p_sigma, e_ps[j]), (new.p_c[b], o.p_c, e_pc[j]),
                            (new.sigma[b], o.sigma, e_sigma[j]), (new.C[b], o.C, e_C[j])):
            err = (got.double().cpu() - torch.as_tensor(np.asarray(ref, dtype=np.float64))).abs()
            bound = 2 * e.cpu() + 1e-30
            q = torch.where(torch.isfinite(err), err / bound, torch.full_like(err, float("inf")))
            r = max(r, float(q.max()))
        ratios.append(r)
    return ratios
