"""The functional XNES and SNES tells for a batch of independent searches, restated item by item on the numpy oracle of the
object-API updates (es_oracle: the ranking, `grad_exp_gaussian` / `update_exp_gaussian` with its float64 matrix exponential,
`grad_exp_separable` / `update_distribution`).  Items are (B, ...) arrays; every item has its own centre, factor or stdev."""

from __future__ import annotations

import numpy as np

from . import es_oracle as E


def xnes_tell(mu, A, A_inv, X, f, *, maximize: bool, ranking: str, lr_mu: float, lr_A: float) -> tuple:
    """(mu', A', A_inv') of every item: z = A_inv (x - mu), utilities centred unless `ranking` is "centered" / "normalized",
    d = sum w z, M = sum w z z^T - (sum w) I, mu' = mu + A (lr_mu d), A' = A expm(lr_A M / 2), A_inv' = expm(-lr_A M / 2) A_inv."""
    out = [], [], []
    for b in range(len(mu)):
        w = E.rank(f[b], ranking, maximize)
        g = E.grad_exp_gaussian(X[b], w, mu[b], A_inv[b], ranking)
        for acc, v in zip(out, E.update_exp_gaussian(mu[b], A[b], A_inv[b], g, lr_mu, lr_A)):
            acc.append(v)
    return tuple(np.stack(v) for v in out)


def snes_tell(mu, sigma, X, f, *, maximize: bool, ranking: str, lr_mu: float, lr_sigma: float, stdev_min=None, stdev_max=None,
              stdev_max_change=None) -> tuple:
    """(mu', sigma') of every item: utilities divided by sum |w| unless `ranking` is "nes", grad_mu = sum w (x - mu),
    grad_sigma = sum w (((x - mu) / sigma)^2 - 1), mu' = mu + lr_mu grad_mu, sigma' = sigma exp(lr_sigma grad_sigma / 2) clamped
    against sigma to the bounds."""
    mus, sigmas = [], []
    for b in range(len(mu)):
        w = E.rank(f[b], ranking, maximize)
        g = E.grad_exp_separable(X[b], w, mu[b], sigma[b], ranking)
        m1, s1 = E.update_distribution(mu[b], sigma[b], g, exp_sigma=True, lr_mu=lr_mu, lr_sigma=lr_sigma, stdev_min=stdev_min,
                                       stdev_max=stdev_max, stdev_max_change=stdev_max_change)
        mus.append(m1)
        sigmas.append(s1)
    return np.stack(mus), np.stack(sigmas)


def expm_pair(S) -> tuple:
    """(expm(S) - I, expm(-S) - I) in float64 for every matrix of S (B, D, D)."""
    S = np.asarray(S, dtype=np.float64)
    eye = np.eye(S.shape[-1])
    return np.stack([E._expm(s) - eye for s in S]), np.stack([E._expm(-s) - eye for s in S])
