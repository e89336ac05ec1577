"""numpy restatement of FSA's predictive gradients with respect to the test inputs, on top of xgrad_oracle's input
derivatives (cov_dx, kdiag_dx, mean_dx) and fsa_oracle.fsa_fit."""
import numpy as np
import scipy.linalg as sl

from oracle import gp_oracle as orc
from xgrad_oracle import cov_dx, kdiag_dx, mean_dx


def fsa_predict_f_grad(spec, X, Xu, f, Xs, blockindpred, mspec=("MeanZero",)):
    """(mu, var, dmu, dvar) of FSA's predict_f(gp, x, blockindpred) (full_scale_approximation.jl:413-478) from
    fsa_oracle.fsa_fit, point by point.  With c = Lambda_xf row m (0 unless test block j holds m and training block j is
    non-empty), h = Lambda_b^-1 c', r = k_u - K_ub h, s = S^-1 r (S = Sigma_QR) and D_u, D_b the input derivatives of
    k(x*, Xu) and k(x*, X_b):
        mu = m(x*) + k_u u + c alpha_b ,     var = k** - k_u' K_uu^-1 k_u - c h + r' s
        dmu  = D_u (u - K_uu^-1 K_ub alpha_b) + D_b alpha_b + dm/dx*
        dvar = dk(x*, x*)/dx* + D_u (2 s - 2 K_uu^-1 k_u - K_uu^-1 K_ub e) + D_b e ,   e = -2 Lambda_b^-1 (c' + K_bu s)
    var is not clamped."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xs = np.ascontiguousarray(Xs, dtype=np.float64)
    Ms = Xs.shape[0]
    blocks, Ulam, Uuu, Us = f["blocks"], f["Ulam"], f["Uuu"], f["Us"]
    pair = np.full(Ms, -1, dtype=np.int64)
    for j, ind in enumerate(blockindpred):
        if j < len(blocks) and blocks[j].size:
            pair[np.asarray(ind, dtype=np.int64)] = j
    Ksu, Du = cov_dx(spec, Xs, Xu)
    Kuf = orc.cov(spec, Xu, X)
    mx, _ = orc.mean_and_grads(mspec, Xs)
    kss = np.diag(orc.cov(spec, Xs, Xs))
    u, alpha = f["alpha_u"], f["alpha"]
    mu = mx + Ksu @ u
    var = np.empty(Ms)
    dmu = np.einsum("mjp,j->mp", Du, u) + mean_dx(mspec, Xs)
    dvar = kdiag_dx(spec, Xs)
    for m in range(Ms):
        ku = Ksu[m]
        Kinv_ku = sl.cho_solve((Uuu, False), ku)
        b = pair[m]
        if b < 0:
            s = sl.cho_solve((Us, False), ku)
            var[m] = kss[m] - ku @ Kinv_ku + ku @ s
            dvar[m] += Du[m].T @ (2.0 * s - 2.0 * Kinv_ku)
            continue
        ind = blocks[b]
        Kub = Kuf[:, ind]
        Kinv_Kub = sl.cho_solve((Uuu, False), Kub)
        kb, Db = cov_dx(spec, Xs[m:m + 1], X[ind])
        c = kb[0] - ku @ Kinv_Kub
        h = sl.cho_solve((Ulam[b], False), c)
        r = ku - Kub @ h
        s = sl.cho_solve((Us, False), r)
        ab = alpha[ind]
        mu[m] += c @ ab
        var[m] = kss[m] - ku @ Kinv_ku - c @ h + r @ s
        e = -2.0 * sl.cho_solve((Ulam[b], False), c + Kub.T @ s)
        dmu[m] += Db[0].T @ ab - Du[m].T @ (Kinv_Kub @ ab)
        dvar[m] += Du[m].T @ (2.0 * s - 2.0 * Kinv_ku - Kinv_Kub @ e) + Db[0].T @ e
    return mu, var, dmu, dvar
