"""Dense numpy restatement of the gradients with respect to the training inputs X (N, d).

GPE: mll = -1/2 r'K^-1 r - 1/2 log|K| - N/2 log 2pi, r = y - m(X).  With A = alpha alpha' - K^-1, dmll = 1/2 sum_ij A_ij dK_ij,
and x_i enters row i (first argument) and column i (second argument) of K, k(a, b) = k(b, a):

    dmll/dx_i = sum_j A_ij d1k(x_i, x_j) + alpha_i dm(x_i)/dx_i

The j = i term is the one-sided partial d1k(x_i, x_i), half of d/dx k(x, x): non-zero for Lin / Poly, the limit 0 for the
stationary leaves (xgrad_oracle.cov_dx).  Noise terms (sigma^2, per-point noise, the Noise leaf) contribute nothing.

GPA (f = L v + m(X), v fixed): the reverse pass through the Cholesky factor is 1/2 sum S dK (gpa_oracle.S_closed), so

    dtarget/dx_i = sum_j S_ij d1k(x_i, x_j) + (dl_df)_i dm(x_i)/dx_i

fd_* are fourth-order central differences of the oracles' mll / target in every coordinate of X."""
import numpy as np

from oracle import gp_oracle as orc
import gpa_oracle as go
from xgrad_oracle import cov_dx, mean_dx


def contract(spec, X, A):
    """sum_j A_ij d1k(x_i, x_j) for a symmetric A (N, N): the device's grad_inputs"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    _, D = cov_dx(spec, X, X)
    return np.einsum("ij,ijp->ip", A, D)


def dmll_dx(spec, X, y, log_noise, mspec=("MeanZero",)):
    """(N, d) gradient of the GPE mll with respect to X"""
    f = orc.mll_and_dmll(spec, X, y, log_noise, mspec)
    return contract(spec, X, f["A"]) + f["alpha"][:, None] * mean_dx(mspec, X)


def dtarget_dx(spec, X, y, mspec, lik, v):
    """(N, d) gradient of the GPA target at fixed v with respect to X"""
    o = go.update_dll(spec, X, y, mspec, lik, v)
    S = go.S_closed(o["L"], o["g"], v)
    return contract(spec, X, S) + o["g"][:, None] * mean_dx(mspec, X)


def _fd(fun, X, h):
    X = np.array(X, dtype=np.float64)
    g = np.zeros_like(X)
    for i in range(X.shape[0]):
        for p in range(X.shape[1]):
            vals = []
            for s in (2, 1, -1, -2):
                Xp = X.copy()
                Xp[i, p] += s * h
                vals.append(fun(Xp))
            g[i, p] = (-vals[0] + 8 * vals[1] - 8 * vals[2] + vals[3]) / (12 * h)
    return g


def fd_dmll_dx(spec, X, y, log_noise, mspec=("MeanZero",), h=1e-3):
    return _fd(lambda Xp: orc.fit(spec, Xp, y, log_noise, mspec)["mll"], X, h)


def fd_dtarget_dx(spec, X, y, mspec, lik, v, h=1e-3):
    return _fd(lambda Xp: go.update_target(spec, Xp, y, mspec, lik, v)["target"], X, h)
