"""Dense restatement of cross-validation on the sparse covariances (FITC, DTC, SoR) for the tests.

Sigma is the matrix `oracle.gp_oracle.fitc_fit` returns (the covariance the engine's mll inverts); its derivatives are built
densely from the kernel derivatives:
    Sigma   = Lambda + Q,  Q = K_fu K_uu^-1 K_uf,  Lambda = sigma^2 + diag(K_ff - Q) (FITC) or sigma^2 (DTC, SoR)
    dQ_j    = dK_fu K_uu^-1 K_uf + K_fu K_uu^-1 dK_uf - K_fu K_uu^-1 dK_uu K_uu^-1 K_uf
    dSigma_j = dQ_j + diag(dk_ii - dQ_j,ii) (FITC) or dQ_j (DTC, SoR);  d Sigma / d sigma^2 = I
(the K_uu nuggets are constants).  The per-parameter bodies of the oracle's literal cross-validation restatement
(`_loo_component`, `_fold_component`) are then fed inv(Sigma), alpha and Z_j = inv(Sigma) dSigma_j; the value functions
(`predict_loo`, `logp_loo`, `predict_cvfold`, `logp_cvfold`) take a dict with U = chol(Sigma)."""
import math

import numpy as np

from oracle import gp_oracle as orc


def sigma_and_grads(spec, X, Xu, log_noise, mode="FITC"):
    """(Sigma, [dSigma_j over the kernel's full parameter vector]) -- nuggets as in fitc_fit"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xu = np.ascontiguousarray(Xu, dtype=np.float64)
    n, m = X.shape[0], Xu.shape[0]
    Kuu, gKuu = orc.cov_and_grads(spec, Xu, None, True)
    Kuu = Kuu + 1e-10 * np.eye(m)
    Kuf, gKuf = orc.cov_and_grads(spec, Xu, X, True)
    A = np.linalg.solve(Kuu, Kuf)                                  # K_uu^-1 K_uf
    Q = Kuf.T @ A
    kdiag = orc._kdiag(spec, X)
    gdiag = [np.array([orc.cov_and_grads(spec, X[i:i + 1], X[i:i + 1], True)[1][p][0, 0] for i in range(n)])
             for p in range(len(gKuu))]
    s2 = math.exp(2.0 * log_noise)
    lam = s2 + kdiag - np.diag(Q) if mode == "FITC" else np.full(n, s2)
    Sigma = Q + np.diag(lam)
    grads = []
    for p in range(len(gKuu)):
        B = gKuf[p].T @ A
        dQ = B + B.T - A.T @ gKuu[p] @ A
        if mode == "FITC":
            dQ = dQ + np.diag(gdiag[p] - np.diag(dQ))
        grads.append(dQ)
    return Sigma, grads


def cv_dict(Sigma, alpha):
    """the dict the oracle's value functions read: U = chol(Sigma) (upper), alpha"""
    return dict(U=np.linalg.cholesky(Sigma).T.copy(), alpha=np.asarray(alpha, dtype=np.float64))


def cv_vectors(invS, dSigma, alpha):
    """(Z_j alpha, diag(Z_j inv(Sigma))) for Z_j = inv(Sigma) dSigma"""
    Z = invS @ dSigma
    return Z @ alpha, np.einsum("ij,ji->i", Z, invS)


def dlogp_loo(Sigma, grads, alpha, y, log_noise, noise=True, kern=True, params=None):
    """dlogpdθ_LOO (crossvalidation.jl:150-178) with dSigma_j in place of dK_j: [noise; kernel parameters `params`]"""
    invS = np.linalg.inv(Sigma)
    out = []
    if noise:
        out.append(-orc._loo_component(invS, alpha, y, invS) / 2.0 * 2.0 * math.exp(2.0 * log_noise))
    if kern:
        for p in (range(len(grads)) if params is None else params):
            out.append(-0.5 * orc._loo_component(invS, alpha, y, invS @ grads[p]))
    return np.array(out)


def dlogp_cvfold(Sigma, grads, alpha, y, log_noise, folds, noise=True, kern=True, params=None):
    """dlogpdθ_CVfold (crossvalidation.jl:264-341) with dSigma_j in place of dK_j"""
    invS = np.linalg.inv(Sigma)
    out = []

    def comp(Z):
        return sum(orc._fold_component(invS, alpha, Z @ invS, Z @ alpha, V) for V in folds)
    if noise:
        out.append(-comp(invS) / 2.0 * 2.0 * math.exp(2.0 * log_noise))
    if kern:
        for p in (range(len(grads)) if params is None else params):
            out.append(-0.5 * comp(invS @ grads[p]))
    return np.array(out)
