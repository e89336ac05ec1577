"""Dense numpy restatement of the predictive gradients with respect to the test inputs.

cov_dx(spec, X1, X2) gives K(X1, X2) and D[a, b, p] = dk(x1_a, x2_b)/dx1_{a,p} for every kernel leaf, Sum, Prod, Masked and
Fixed, in the spec format of oracle/gp_oracle.py.  predict_f_grad gives (mu, var, dmu, dvar) of the dense prediction
(GP.jl:25-79) from gp_oracle.fit:

    dmu[m, p]  = sum_i D(x*, X)[m, i, p] alpha_i + dmean/dx*_{m,p}
    dvar[m, p] = 2 D(x*_m, x*_m)[p] - 2 sum_i D(x*, X)[m, i, p] (K^-1 k*_m)_i

Where a test point coincides with an input (r = 0) the stationary leaves give the limit of the derivative, 0; Mat12, whose
derivative does not exist there, also gives 0.  var is not clamped here."""
import math

import numpy as np
import scipy.linalg as sl

from oracle import gp_oracle as orc


def _leaf_dx(name, theta, extra, X1, X2):
    th = [float(t) for t in theta]
    K, _ = orc._leaf(name, theta, extra, X1, X2, False)
    diff = X1[:, None, :] - X2[None, :, :]
    n1, n2, d = diff.shape
    r2 = np.sum(diff * diff, axis=2)
    with np.errstate(divide="ignore", invalid="ignore"):
        if name == "SEIso":
            return K, -(K / math.exp(2 * th[0]))[..., None] * diff
        if name in ("SEArd", "Mat12Ard", "Mat32Ard", "Mat52Ard", "RQArd"):
            nw = d
            il2 = np.exp(-2.0 * np.array(th[:nw]))
            wr2 = np.sum(diff * diff * il2, axis=2)
            if name == "SEArd":
                f = -K
            elif name == "RQArd":
                s2, al = math.exp(2 * th[-2]), math.exp(th[-1])
                f = -s2 * (1 + wr2 / (2 * al)) ** (-al - 1)
            else:
                s2, r = math.exp(2 * th[-1]), np.sqrt(wr2)
                if name == "Mat12Ard":
                    f = np.where(r > 0, -s2 * np.exp(-r) / r, 0.0)
                elif name == "Mat32Ard":
                    f = -3.0 * s2 * np.exp(-math.sqrt(3.0) * r)
                else:
                    s = math.sqrt(5.0) * r
                    f = -5.0 / 3.0 * s2 * (1 + s) * np.exp(-s)
            return K, f[..., None] * diff * il2
        if name in ("Mat12Iso", "Mat32Iso", "Mat52Iso"):
            l, s2, r = math.exp(th[0]), math.exp(2 * th[1]), np.sqrt(r2)
            if name == "Mat12Iso":
                f = np.where(r > 0, -K / (l * r), 0.0)
            elif name == "Mat32Iso":
                f = -3.0 * s2 * np.exp(-math.sqrt(3.0) * r / l) / l ** 2
            else:
                s = math.sqrt(5.0) * r / l
                f = -5.0 / 3.0 * s2 * (1 + s) * np.exp(-s) / l ** 2
            return K, f[..., None] * diff
        if name == "RQIso":
            l2, s2, al = math.exp(2 * th[0]), math.exp(2 * th[1]), math.exp(th[2])
            f = -s2 * (1 + r2 / (2 * al * l2)) ** (-al - 1) / l2
            return K, f[..., None] * diff
        if name == "Periodic":
            l2, per = math.exp(2 * th[0]), math.exp(th[2])
            r = np.sqrt(r2)
            u = math.pi * r / per
            s2r = np.where(r > 0, np.sin(2 * u) / r, 2 * math.pi / per)
            f = -K * (2.0 / l2) * (math.pi / per) * s2r
            return K, f[..., None] * diff
    if name == "LinIso":
        return K, np.broadcast_to(X2[None, :, :] / math.exp(2 * th[0]), diff.shape).copy()
    if name == "LinArd":
        l = np.exp(np.array(th))
        return K, np.broadcast_to(X2[None, :, :] / l ** 2, diff.shape).copy()
    if name == "Poly":
        c, s2, deg = math.exp(th[0]), math.exp(2 * th[1]), int(extra)
        base = c + orc._dot(X1, X2)
        f = s2 * deg * base ** (deg - 1) if deg >= 1 else np.zeros_like(base)
        return K, f[..., None] * X2[None, :, :]
    if name in ("Noise", "Const"):
        return K, np.zeros(diff.shape)
    raise ValueError("unknown kernel leaf %r" % (name,))


def cov_dx(spec, X1, X2):
    """(K, D): K[a, b] = k(x1_a, x2_b), D[a, b, p] = dk(x1_a, x2_b)/dx1_{a,p}."""
    X1 = np.ascontiguousarray(X1, dtype=np.float64)
    X2 = np.ascontiguousarray(X2, dtype=np.float64)
    name = spec[0]
    if name in ("Sum", "Prod"):
        Kl, Dl = cov_dx(spec[1], X1, X2)
        Kr, Dr = cov_dx(spec[2], X1, X2)
        if name == "Sum":
            return Kl + Kr, Dl + Dr
        return Kl * Kr, Dl * Kr[..., None] + Kl[..., None] * Dr
    if name == "Masked":
        dims = list(spec[2])
        K, Dm = cov_dx(spec[1], X1[:, dims], X2[:, dims])
        D = np.zeros((X1.shape[0], X2.shape[0], X1.shape[1]))
        D[:, :, dims] = Dm
        return K, D
    if name == "Fixed":
        return cov_dx(spec[1], X1, X2)
    extra = spec[2] if len(spec) > 2 else None
    return _leaf_dx(name, spec[1], extra, X1, X2)


def kdiag_dx(spec, Xs):
    """d k(x, x)/dx at every row of Xs (M, d): 2 dk(x, x')/dx at x' = x, every kernel being symmetric."""
    D = np.stack([cov_dx(spec, Xs[m:m + 1], Xs[m:m + 1])[1][0, 0] for m in range(Xs.shape[0])])
    return 2.0 * D


def mean_dx(mspec, Xs):
    if mspec[0] == "MeanLin":
        return np.broadcast_to(np.asarray(mspec[1], dtype=np.float64), Xs.shape).copy()
    return np.zeros(Xs.shape)


def predict_f_grad(spec, X, f, Xs, mspec=("MeanZero",), alpha=None):
    """(mu, var, dmu, dvar) of the dense prediction; dmu / dvar are (M, d).  f = gp_oracle.fit(...); alpha defaults to f's."""
    Xs = np.ascontiguousarray(Xs, dtype=np.float64)
    alpha = f["alpha"] if alpha is None else alpha
    Kc, D = cov_dx(spec, Xs, X)                                     # M x N, M x N x d
    mx, _ = orc.mean_and_grads(mspec, Xs)
    mu = mx + Kc @ alpha
    V = sl.solve_triangular(f["U"], Kc.T, trans="T", lower=False)
    var = np.diag(orc.cov(spec, Xs, Xs)) - np.sum(V * V, axis=0)
    W = sl.solve_triangular(f["U"], V, lower=False)                 # K^-1 K*'  (N x M)
    dmu = np.einsum("mip,i->mp", D, alpha) + mean_dx(mspec, Xs)
    dvar = kdiag_dx(spec, Xs) - 2.0 * np.einsum("mip,im->mp", D, W)
    return mu, var, dmu, dvar


def fitc_predict_f_grad(spec, X, Xu, f, Xs, mspec=("MeanZero",)):
    """(mu, var, dmu, dvar) of the FITC / DTC / SoR prediction (fitc.jl:324-332 -> dtc.jl:41-59 -> sor.jl:302-321) from
    gp_oracle.fitc_fit: mu = mx + K*u alpha_u, var = k** - |L_uu^-1 k_u*|^2 + |L_s^-1 k_u*|^2 (SoR: the last term only), so
    dvar = 2c dk(x*, x*)/dx* - 2 sum_j dk(x*, u_j)/dx* W[m, j] with W = K*u K_uu^-1 - K*u Sigma_QR^-1 (SoR: c = 0, no K_uu^-1
    term).  var is not clamped."""
    Xs = np.ascontiguousarray(Xs, dtype=np.float64)
    Ksu, D = cov_dx(spec, Xs, Xu)                                   # M x Mu, M x Mu x d
    mx, _ = orc.mean_and_grads(mspec, Xs)
    mu = mx + Ksu @ f["alpha_u"]
    A = sl.solve_triangular(f["Uuu"], Ksu.T, trans="T", lower=False)
    B = sl.solve_triangular(f["Us"], Ksu.T, trans="T", lower=False)
    Wb = sl.solve_triangular(f["Us"], B, lower=False)               # Sigma_QR^-1 K_u*
    dmu = np.einsum("mjp,j->mp", D, f["alpha_u"]) + mean_dx(mspec, Xs)
    if f.get("mode", "FITC") == "SoR":
        var = np.sum(B * B, axis=0)
        dvar = 2.0 * np.einsum("mjp,jm->mp", D, Wb)
        return mu, var, dmu, dvar
    Wa = sl.solve_triangular(f["Uuu"], A, lower=False)              # K_uu^-1 K_u*
    var = np.diag(orc.cov(spec, Xs, Xs)) - np.sum(A * A, axis=0) + np.sum(B * B, axis=0)
    dvar = kdiag_dx(spec, Xs) - 2.0 * np.einsum("mjp,jm->mp", D, Wa - Wb)
    return mu, var, dmu, dvar
