"""Dense numpy restatement of dmll/dX, the gradient of the sparse mll with respect to the training inputs, for FITC, DTC,
SoR and FSA.

The mll is exactly the one oracle/gp_oracle.fitc_fit and tests/fsa_oracle.fsa_fit compute, nuggets included; in the form
of inducing_grad_oracle,

    mll = -1/2 [ r' S^-1 r + logdet S + logdet K2 - logdet K1 + N log 2 pi ],   S = Lambda + K_fu K2^-1 K_uf,  r = y - m(X)

with K1 = K_uu + 1e-10 I, K2 = K_uu + 2e-10 I and Lambda = sigma^2 + diag(K_ff - K_fu K1^-1 K_uf) (FITC), sigma^2 I (DTC,
SoR) or blockdiag(K_bb - K_bu K1^-1 K_ub) + (sigma^2 + 1e-10) I (FSA).  K_uu does not depend on X.  With A = alpha alpha' -
S^-1, B1 = K1^-1 K_uf, B2 = K2^-1 K_uf and Gd the part of A that Lambda sees (diag(A) for FITC, the diagonal blocks of A
for FSA, 0 for DTC / SoR):

    dmll = 1/2 <G_uf, dK_uf> + 1/2 <Gd, dK_ff>,   G_uf = 2 B2 A - 2 B1 Gd       (inducing_grad_oracle's G_uf)

x_i enters column i of K_uf and row and column i of K_ff, so with d1k the derivative in the first argument (k symmetric)

    dmll/dx_i = 1/2 [ sum_j G_uf[j, i] d1k(x_i, u_j) + sum_l (Gd[i, l] + Gd[l, i]) d1k(x_i, x_l) ] + alpha_i dm(x_i)/dx_i

-- for FITC the second sum is 2 Gd_ii d1k(x_i, x_i), the derivative of k(x_i, x_i) weighted by g_i = Gd_ii; for FSA it runs
over the block of i.  At coincident points the stationary leaves give the limit of d1k, 0 (xgrad_oracle.cov_dx).
S is formed densely: small N only (a few thousand)."""
import numpy as np

from oracle import gp_oracle as orc
from inducing_grad_oracle import MODES, fit, mll
import xgrad_oracle as xo

__all__ = ["MODES", "dmll_dx", "fd_dmll_dx", "fit", "mll"]


def adjoints(spec, X, Xu, y, log_noise, mode, blocks=None, mspec=("MeanZero",)):
    """(G_uf (M, N), Gd (N, N), alpha (N,)) of the dense restatement"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xu = np.ascontiguousarray(Xu, dtype=np.float64)
    n, m = X.shape[0], Xu.shape[0]
    sig2 = np.exp(2.0 * log_noise)
    Kraw = orc.cov(spec, Xu)
    Kuf = orc.cov(spec, Xu, X)
    K1i = np.linalg.inv(Kraw + 1e-10 * np.eye(m))
    K2i = np.linalg.inv(Kraw + 2e-10 * np.eye(m))
    B1, B2 = K1i @ Kuf, K2i @ Kuf
    if mode == "FITC":
        Lam = np.diag(sig2 + orc._kdiag(spec, X) - np.sum(Kuf * B1, axis=0))
    elif mode in ("DTC", "SoR"):
        Lam = sig2 * np.eye(n)
    elif mode == "FSA":
        Lam = np.zeros((n, n))
        for ind in blocks:
            ind = np.asarray(ind, dtype=np.int64)
            if ind.size:
                Lam[np.ix_(ind, ind)] = orc.cov(spec, X[ind]) - Kuf[:, ind].T @ B1[:, ind] + (sig2 + 1e-10) * np.eye(ind.size)
    else:
        raise ValueError("unknown mode %r" % (mode,))
    Si = np.linalg.inv(Lam + Kuf.T @ B2)
    Si = (Si + Si.T) / 2.0
    r = np.asarray(y, dtype=np.float64) - orc.mean_and_grads(mspec, X)[0]
    alpha = Si @ r
    A = np.outer(alpha, alpha) - Si
    Gd = np.zeros((n, n))
    if mode == "FITC":
        Gd = np.diag(np.diag(A))
    elif mode == "FSA":
        for ind in blocks:
            ind = np.asarray(ind, dtype=np.int64)
            Gd[np.ix_(ind, ind)] = A[np.ix_(ind, ind)]
    return 2.0 * B2 @ A - 2.0 * B1 @ Gd, Gd, alpha


def dmll_dx(spec, X, Xu, y, log_noise, mode, blocks=None, mspec=("MeanZero",)):
    """dmll/dX as an (N, d) array, point-major (one training point per row), the mean's part included"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Guf, Gd, alpha = adjoints(spec, X, Xu, y, log_noise, mode, blocks, mspec)
    _, Dfu = xo.cov_dx(spec, X, Xu)                              # N x M x d, derivative in x_i
    g = np.einsum("ji,ijp->ip", Guf, Dfu)
    if np.any(Gd):
        _, Dff = xo.cov_dx(spec, X, X)                           # N x N x d, derivative in the first argument
        g += np.einsum("il,ilp->ip", Gd + Gd.T, Dff)
    return 0.5 * g + alpha[:, None] * xo.mean_dx(mspec, X)


def fd_dmll_dx(spec, X, Xu, y, log_noise, mode, blocks=None, mspec=("MeanZero",), h=1e-3):
    """fourth-order central differences of the oracle mll in every coordinate of X, (N, d)"""
    X = np.asarray(X, dtype=np.float64)
    out = np.empty(X.shape)
    for i in range(X.shape[0]):
        for p in range(X.shape[1]):
            f = []
            for s in (-2, -1, 1, 2):
                Z = X.copy()
                Z[i, p] += s * h
                f.append(mll(spec, Z, Xu, y, log_noise, mode, blocks, mspec))
            out[i, p] = (f[0] - 8.0 * f[1] + 8.0 * f[2] - f[3]) / (12.0 * h)
    return out
