"""Float64 numpy restatement of the transformed objectives the tests use, independent of evotorch_b200.jit.

Every function takes rows X (..., n, D) and a transform M (..., D, D), o (..., D) whose batch dimensions broadcast against
those of X, and returns the fitnesses (..., n).  y = M (x - o) per row: y_j = sum_k M[j, k] (x_k - o_k).
"""

import numpy as np


def transformed(X, M, o):
    X, M, o = (np.asarray(a, np.float64) for a in (X, M, o))
    return np.einsum("...jk,...nk->...nj", M, X - o[..., None, :])


def _weights(D):
    return 10.0 ** (6.0 * np.arange(D) / max(D - 1, 1))


def rot_ellipsoid(X, M, o):
    """sum_j 10^(6 j / max(D - 1, 1)) y_j^2: condition 1e6."""
    y = transformed(X, M, o)
    return (_weights(y.shape[-1]) * y**2).sum(-1)


def rot_rastrigin(X, M, o):
    y = transformed(X, M, o)
    return 10.0 * y.shape[-1] + (y**2 - 10.0 * np.cos(2 * np.pi * y)).sum(-1)


def rot_rosenbrock(X, M, o):
    """sum_{j < D-1} 100 (y_{j+1} - y_j^2)^2 + (1 - y_j)^2 (0 at D = 1)."""
    y = transformed(X, M, o)
    return (100.0 * (y[..., 1:] - y[..., :-1] ** 2) ** 2 + (1.0 - y[..., :-1]) ** 2).sum(-1)


def rot_schwefel_1_2(X, M, o):
    y = transformed(X, M, o)
    return (np.cumsum(y, -1) ** 2).sum(-1)


def lunacek_like(X, M, o, sg, mu1, s):
    """BBOB f24's structure: the bi-sphere on x_hat = 2 sg x, the Rastrigin cosine on y, and the boundary penalty on x.  sg (..., D),
    mu1 and s (..., 1) broadcast like M and o.  minimum and maximum ignore a NaN operand, as the language's do (fmin / fmax)."""
    X = np.asarray(X, np.float64)
    y = transformed(X, M, o)
    sg, mu1, s = (np.asarray(a, np.float64)[..., None, :] for a in (sg, mu1, s))
    D = X.shape[-1]
    a = ((2 * sg * X - 2.5) ** 2).sum(-1)
    b = ((2 * sg * X - mu1) ** 2).sum(-1)
    c = np.cos(2 * np.pi * y).sum(-1)
    p = (np.fmax(0.0, np.abs(X) - 5.0) ** 2).sum(-1)
    return np.fmin(a, D + s[..., 0] * b) + 10.0 * (D - c) + 1e4 * p


def penalised_ellipsoid(X, M, o):
    """The rotated ellipsoid plus BBOB's boundary penalty 100 sum max(0, |x_j| - 5)^2 on x, without noise."""
    X = np.asarray(X, np.float64)
    return rot_ellipsoid(X, M, o) + 100.0 * (np.fmax(0.0, np.abs(X) - 5.0) ** 2).sum(-1)
