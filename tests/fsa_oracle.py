"""CPU oracle of the Full Scale Approximation (src/sparse/full_scale_approximation.jl), restated block by block with
numpy on top of oracle/gp_oracle.py's kernels: b x b blocks and M x N matrices only, so it runs at N = 70 000.  The
dense N x N Sigma is built only for N <= 4096 (as gp_oracle.fitc_fit does)."""
import math

import numpy as np
import scipy.linalg as sl

from oracle.gp_oracle import LOG2PI, _potrf_upper, _potrs_upper, cov, cov_and_grads, mean_and_grads


def fsa_fit(spec, X, Xu, blocks, y, log_noise, mspec=("MeanZero",)):
    """update_cK!(::FullScalePDMat) (:197-230), `\\` (:105-108), logdet (:142), dmll_noise (:328-363), get_alpha_u
    (:366-373) and the mll (GPE.jl:210).  blocks: list of 0-based index arrays partitioning 0..N-1."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xu = np.ascontiguousarray(Xu, dtype=np.float64)
    n, m = X.shape[0], Xu.shape[0]
    sig2 = math.exp(2 * log_noise)
    Kuu = cov(spec, Xu) + 1e-10 * np.eye(m)                     # make_posdef!(Kuubuffer; nugget=1e-10)  :204-205
    Uuu = _potrf_upper(Kuu)
    Kuf = cov(spec, Xu, X)                                      # :207
    blocks = [np.asarray(b, dtype=np.int64) for b in blocks]
    Ulam = []
    LamInvKfu = np.zeros((n, m))                                # Λ \ Kfu, block by block (BlockDiagPDMat `\`, :23-29)
    for ind in blocks:                                          # :213-222
        Kblock = cov(spec, X[ind])
        Qchol = sl.solve_triangular(Uuu, Kuf[:, ind], trans="T", lower=False)     # whiten(Kuu_PD, Kuf[:,ind])
        Lam_i = Kblock - Qchol.T @ Qchol + sig2 * np.eye(ind.size) + 1e-10 * np.eye(ind.size)   # + make_posdef! nugget
        U_i = _potrf_upper(Lam_i) if ind.size else np.zeros((0, 0))
        Ulam.append(U_i)
        if ind.size:
            LamInvKfu[ind] = _potrs_upper(U_i, Kuf[:, ind].T)
    SQR = Kuf @ LamInvKfu + Kuu + 1e-10 * np.eye(m)             # :224-227
    Us = _potrf_upper(SQR)

    def lam_solve(v):
        out = np.zeros_like(v)
        for ind, U_i in zip(blocks, Ulam):
            if ind.size:
                out[ind] = _potrs_upper(U_i, v[ind])
        return out

    mu, MG = mean_and_grads(mspec, X)
    r = np.asarray(y, dtype=np.float64) - mu
    Lk = sl.solve_triangular(Us, Kuf, trans="T", lower=False)   # whiten(ΣQR_PD, Kuf)
    lr = lam_solve(r)
    alpha = lam_solve(r - Lk.T @ (Lk @ lr))                     # :105-108
    logdet_lam = sum(2 * np.sum(np.log(np.diag(U_i))) for U_i in Ulam)
    logdet = 2 * np.sum(np.log(np.diag(Us))) - 2 * np.sum(np.log(np.diag(Uuu))) + logdet_lam   # :142
    mll = -(r @ alpha + logdet + LOG2PI * n) / 2.0
    trinv_lam = sum(np.sum(sl.solve_triangular(U_i, np.eye(U_i.shape[0]), lower=False) ** 2) for U_i in Ulam)
    LkL = lam_solve(Lk.T)                                       # Λ \ whiten(ΣQR_PD, Kuf)'  :330
    dnoise = sig2 * (alpha @ alpha - trinv_lam + np.sum(LkL * LkL))                             # :339-343
    alpha_u = _potrs_upper(Us, Kuf @ lr)                        # :366-373
    Sigma = None
    if n <= 4096:                                               # Matrix(::FullScalePDMat)  :143-148
        W = sl.solve_triangular(Uuu, Kuf, trans="T", lower=False)
        Sigma = W.T @ W
        for ind, U_i in zip(blocks, Ulam):
            Sigma[np.ix_(ind, ind)] += U_i.T @ U_i
    return dict(alpha=alpha, mll=mll, logdet=logdet, dmll_noise=dnoise, dmll_mean=MG.T @ alpha, alpha_u=alpha_u,
                Uuu=Uuu, Us=Us, Sigma=Sigma, resid=r, blocks=blocks, Ulam=Ulam, Lk=Lk)


def fsa_dmll_kern(spec, X, Xu, f):
    """Kernel-parameter gradient of the FSA mll, restating the reference literally: the SoR part
    dmll_kern!(..., ::SubsetOfRegsStrategy) (subsetofregressors.jl:219-253, precompute! :140-151) with FSA's solve (:105-108), plus the
    per-block part of dmll_kern!(..., ::FullScaleApproxStrat) (:287-317).  `f` = result of fsa_fit."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xu = np.ascontiguousarray(Xu, dtype=np.float64)
    alpha, Uuu, Us, Lk, blocks, Ulam = f["alpha"], f["Uuu"], f["Us"], f["Lk"], f["blocks"], f["Ulam"]
    Kuf, gKuf = cov_and_grads(spec, Xu, X, True)
    _, gKuu = cov_and_grads(spec, Xu, None, True)
    KuuinvKuf = _potrs_upper(Uuu, Kuf)                                   # Kuu⁻¹Kuf             sor.jl:146
    b = _potrs_upper(Uuu, Kuf @ alpha)                                   # Kuu⁻¹KufΣ⁻¹y         sor.jl:147

    def lam_solve(B):
        out = np.zeros_like(B)
        for ind, U_i in zip(blocks, Ulam):
            if ind.size:
                out[ind] = _potrs_upper(U_i, B[ind])
        return out

    def solve_Sigma(B):                                                  # Σ⁻¹B  (:105-108)
        return lam_solve(B - Lk.T @ (Lk @ lam_solve(B)))

    SinvKfu = solve_Sigma(Kuf.T)                                         # Σ⁻¹Kfu               sor.jl:148
    out = []
    for p in range(len(gKuu)):
        dKuu, dKuf = gKuu[p], gKuf[p]
        V = 2 * alpha @ (dKuf.T @ b) - b @ (dKuu @ b)                    # sor.jl:246-247
        T = 2 * np.sum(solve_Sigma(dKuf.T) * KuuinvKuf.T)                # sor.jl:248
        T -= np.sum(SinvKfu.T * (_potrs_upper(Uuu, dKuu) @ KuuinvKuf))   # sor.jl:249
        g = (V - T) / 2.0
        V2 = T2 = 0.0
        for ind, U_i in zip(blocks, Ulam):                               # :293-309
            if not ind.size:
                continue
            dKi = cov_and_grads(spec, X[ind], None, True)[1][p]
            Ai = KuuinvKuf[:, ind]
            dLam = dKi + Ai.T @ dKuu @ Ai - 2 * dKuf[:, ind].T @ Ai      # :299-301
            V2 += alpha[ind] @ (dLam @ alpha[ind])                       # :302
            L = _potrs_upper(U_i, Lk[:, ind].T)                          # Λi⁻¹ whiten(ΣQR_PD, Kui)'  :305-306
            T2 += np.trace(_potrs_upper(U_i, dLam)) - np.sum(L * (dLam @ L))   # trinvAB(pd, ∂Λi) - dot(L, ∂Λi*L)  :307
        out.append(g + (V2 - T2) / 2.0)                                  # :316
    return np.array(out)


def _lam_xf(spec, X, Xu, f, Xs, blockindpred):
    """Λxf = Kxf - Qxf on the zip-paired (test block, training block) pairs, 0 elsewhere (:426-435); Qab = Kau Kuu⁻¹ Kub"""
    Kxu = cov(spec, Xs, Xu)
    Lam = np.zeros((Xs.shape[0], X.shape[0]))
    for pb, tb in zip(blockindpred, f["blocks"]):
        pb = np.asarray(pb, dtype=np.int64)
        if not pb.size or not tb.size:
            continue
        Qxf = Kxu[pb] @ _potrs_upper(f["Uuu"], cov(spec, Xu, X[tb]))
        Lam[np.ix_(pb, tb)] = cov(spec, Xs[pb], X[tb]) - Qxf
    return Lam


def fsa_predict_full(spec, X, Xu, f, Xs, blockindpred, mspec=("MeanZero",)):
    """predictMVN(xpred, blockindpred, ...) (:413-447) literally: mu = m(x) + Kxu alpha_u + Λxf alpha,
    Σ_FSA = Kxx - (Qxf + Λxf) (Σ \\ (Qxf + Λxf)') with the FSA solve (:105-108).  Dense nx x N matrices."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xs = np.ascontiguousarray(Xs, dtype=np.float64)
    blocks, Ulam, Lk = f["blocks"], f["Ulam"], f["Lk"]

    def lam_solve(B):
        out = np.zeros_like(B)
        for ind, U_i in zip(blocks, Ulam):
            if ind.size:
                out[ind] = _potrs_upper(U_i, B[ind])
        return out

    Lxf = _lam_xf(spec, X, Xu, f, Xs, blockindpred)
    Kux = cov(spec, Xu, Xs)
    mx, _ = mean_and_grads(mspec, Xs)
    mu = mx + Kux.T @ f["alpha_u"] + Lxf @ f["alpha"]                       # :439
    A = Kux.T @ _potrs_upper(f["Uuu"], cov(spec, Xu, X)) + Lxf            # Qxf + Λxf  :442-443
    At = A.T
    SinvAt = lam_solve(At - Lk.T @ (Lk @ lam_solve(At)))                   # Ktrain \\ collect(ΛplusQxf')
    return mu, cov(spec, Xs, Xs) - A @ SinvAt                              # :444-445


def fsa_predict_closed(spec, X, Xu, f, Xs, blockindpred, mspec=("MeanZero",)):
    """The closed form the GPU evaluates: with C = Λxf, G = C L_Λ^-T, W = L_Λ^-1 K_fu, V_* = L_uu^-1 K_u*,
    mu = m(x) + K_*u u + C alpha,  Σ = K_** - V_*'V_* - G G' + R R',  R = (K_*u - G W) L_s^-T."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    Xs = np.ascontiguousarray(Xs, dtype=np.float64)
    C = _lam_xf(spec, X, Xu, f, Xs, blockindpred)
    G = np.zeros_like(C)
    Kfu = cov(spec, X, Xu)
    W = np.zeros_like(Kfu)
    for ind, U_i in zip(f["blocks"], f["Ulam"]):
        if ind.size:
            G[:, ind] = sl.solve_triangular(U_i, C[:, ind].T, trans="T", lower=False).T     # C_i U_i^-1  (L_i = U_i')
            W[ind] = sl.solve_triangular(U_i, Kfu[ind], trans="T", lower=False)           # U_i^-T K_fu,i
    Kxu = cov(spec, Xs, Xu)
    Vs = sl.solve_triangular(f["Uuu"], Kxu.T, trans="T", lower=False)
    R = sl.solve_triangular(f["Us"], (Kxu - G @ W).T, trans="T", lower=False)
    mx, _ = mean_and_grads(mspec, Xs)
    mu = mx + Kxu @ f["alpha_u"] + C @ f["alpha"]
    return mu, cov(spec, Xs, Xs) - Vs.T @ Vs - G @ G.T + R.T @ R


def nearest_blocks(X, Xu):
    """blocks by nearest inducing point (test/test_sparse.jl:35-36), 0-based"""
    d2 = ((X[:, None, :] - Xu[None, :, :]) ** 2).sum(axis=2)
    near = np.argmin(d2, axis=1)
    return [np.flatnonzero(near == i) for i in range(Xu.shape[0])]
