"""Dense numpy restatement of dmll/dXu, the gradient of the sparse mll with respect to the inducing inputs, for FITC, DTC,
SoR and FSA.

The mll is exactly the one oracle/gp_oracle.fitc_fit and tests/fsa_oracle.fsa_fit compute, nuggets included.  With
K1 = K_uu + 1e-10 I (make_posdef!) and Sigma_QR = K_uf Lambda^-1 K_fu + K1 + 1e-10 I, Woodbury and the determinant lemma
turn it into

    mll = -1/2 [ r' S^-1 r + logdet S + logdet K2 - logdet K1 + N log 2 pi ],   S = Lambda + K_fu K2^-1 K_uf,  K2 = K_uu + 2e-10 I

with Lambda = sigma^2 + diag(K_ff - K_fu K1^-1 K_uf) (FITC), sigma^2 I (DTC, SoR) or blockdiag(K_bb - K_bu K1^-1 K_ub) +
(sigma^2 + 1e-10) I (FSA).  Only K_uf and K_uu depend on Xu.  With A = alpha alpha' - S^-1, B1 = K1^-1 K_uf,
B2 = K2^-1 K_uf and Gd the part of A that Lambda sees (diag(A) for FITC, the diagonal blocks of A for FSA, 0 for DTC/SoR):

    dmll = 1/2 <G_uf, dK_uf> + 1/2 <G_uu, dK_uu>
    G_uf = 2 B2 A - 2 B1 Gd ,   G_uu = -B2 A B2' + B1 Gd B1' - (K2^-1 - K1^-1)

and moving u_j changes row j of K_uf and row and column j of K_uu, so (k symmetric)

    dmll/du_j = 1/2 [ sum_i G_uf[j, i] dk(u_j, x_i)/du_j + sum_l (G_uu[j, l] + G_uu[l, j]) dk(u_j, u_l)/du_j ]

with dk/du from tests/xgrad_oracle.cov_dx.  S is formed densely: small N only (a few thousand)."""
import numpy as np

from oracle import gp_oracle as orc
import fsa_oracle as fo
import xgrad_oracle as xo

MODES = ("FITC", "DTC", "SoR", "FSA")


def fit(spec, X, Xu, y, log_noise, mode, blocks=None, mspec=("MeanZero",)):
    """the oracle fit of the strategy (gp_oracle.fitc_fit or fsa_oracle.fsa_fit)"""
    if mode == "FSA":
        return fo.fsa_fit(spec, X, Xu, blocks, y, log_noise, mspec)
    return orc.fitc_fit(spec, X, Xu, y, log_noise, mspec, mode=mode)


def mll(spec, X, Xu, y, log_noise, mode, blocks=None, mspec=("MeanZero",)):
    return fit(spec, X, Xu, y, log_noise, mode, blocks, mspec)["mll"]


def dmll_dxu(spec, X, Xu, y, log_noise, mode, blocks=None, mspec=("MeanZero",)):
    """dmll/dXu as an (M, d) array, point-major (one inducing point per row)"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xu = np.ascontiguousarray(Xu, dtype=np.float64)
    n, m = X.shape[0], Xu.shape[0]
    sig2 = np.exp(2.0 * log_noise)
    Kraw, Duu = xo.cov_dx(spec, Xu, Xu)                          # M x M, M x M x d
    Kuf, Duf = xo.cov_dx(spec, Xu, X)                            # M x N, M x N x d
    K1 = Kraw + 1e-10 * np.eye(m)
    K2 = Kraw + 2e-10 * np.eye(m)
    K1i, K2i = np.linalg.inv(K1), np.linalg.inv(K2)
    B1, B2 = K1i @ Kuf, K2i @ Kuf
    if mode == "FITC":
        kdiag = orc._kdiag(spec, X)
        Lam = np.diag(sig2 + kdiag - np.sum(Kuf * B1, axis=0))
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
    S = Lam + Kuf.T @ B2
    r = np.asarray(y, dtype=np.float64) - orc.mean_and_grads(mspec, X)[0]
    Si = np.linalg.inv(S)
    Si = (Si + Si.T) / 2.0
    alpha = Si @ r
    A = np.outer(alpha, alpha) - Si
    if mode == "FITC":
        Gd = np.diag(np.diag(A))
    elif mode == "FSA":
        Gd = np.zeros((n, n))
        for ind in blocks:
            ind = np.asarray(ind, dtype=np.int64)
            Gd[np.ix_(ind, ind)] = A[np.ix_(ind, ind)]
    else:
        Gd = np.zeros((n, n))
    Guf = 2.0 * B2 @ A - 2.0 * B1 @ Gd
    Guu = -B2 @ A @ B2.T + B1 @ Gd @ B1.T - (K2i - K1i)
    Wuu = Guu + Guu.T
    return 0.5 * (np.einsum("jip,ji->jp", Duf, Guf) + np.einsum("jlp,jl->jp", Duu, Wuu))


def fd_dmll_dxu(spec, X, Xu, y, log_noise, mode, blocks=None, h=1e-3):
    """fourth-order central differences of the oracle mll in every coordinate of Xu, (M, d).  The step is large because
    the mll carries the rounding of cond(Sigma_QR) (1e7 in some zoo cases); the truncation error is O(h^4)."""
    Xu = np.asarray(Xu, dtype=np.float64)
    out = np.empty(Xu.shape)
    for j in range(Xu.shape[0]):
        for p in range(Xu.shape[1]):
            f = []
            for s in (-2, -1, 1, 2):
                U = Xu.copy()
                U[j, p] += s * h
                f.append(mll(spec, X, U, y, log_noise, mode, blocks))
            out[j, p] = (f[0] - 8.0 * f[1] + 8.0 * f[2] - f[3]) / (12.0 * h)
    return out


def conditioning(spec, X, Xu, log_noise, mode, blocks=None):
    """(cond(K_uu + 1e-10 I), cond(Sigma_QR)) of the oracle fit, printed beside device errors"""
    f = fit(spec, X, Xu, np.zeros(X.shape[0]), log_noise, mode, blocks)
    c1 = np.linalg.cond(f["Uuu"]) ** 2
    c2 = np.linalg.cond(f["Us"]) ** 2
    return c1, c2
