"""CPU oracle of GPA (src/GPA.jl, src/likelihoods/*.jl, src/chol_utils.jl), restated literally with numpy on top of
oracle/gp_oracle.py's kernels and means.  Likelihoods are tuples: ("BernLik",), ("BinLik", n), ("ExpLik",),
("GaussLik", lσ), ("PoisLik",), ("StuTLik", ν, lσ).  The reverse-mode Cholesky is ported loop for loop (O(N^3) level-2
steps); `update_dll(..., method="closed")` uses the closed form the device computes (S = W' M_s W), for sizes where the
loop is too slow."""
import math

import numpy as np
import scipy.linalg as sl
from scipy.special import gammaln

from oracle.gp_oracle import LOG2PI, cov, cov_and_grads, mean_and_grads


def _Phi(x):                               # StatsFuns normcdf
    return 0.5 * math.erfc(-x / math.sqrt(2.0))


def _phi(x):                               # StatsFuns normpdf
    return math.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# ---- likelihoods -------------------------------------------------------------------------------------------------------
def log_dens(lik, f, y):
    name = lik[0]
    if name == "BernLik":                  # bernoulli.jl:12-14
        return np.array([math.log(_Phi(fi)) if yi else math.log(1.0 - _Phi(fi)) for fi, yi in zip(f, y)])
    if name == "BinLik":                   # binomial.jl:16-19
        n = lik[1]
        th = np.exp(f) / (1 + np.exp(f))
        return np.array([gammaln(n + 1.0) - gammaln(yi + 1.0) - gammaln(n - yi + 1.0) + yi * math.log(ti) + (n - yi) * math.log(1 - ti)
                         for ti, yi in zip(th, y)])
    if name == "ExpLik":                   # exponential.jl:13-16
        return np.array([-fi - math.exp(-fi) * yi for fi, yi in zip(f, y)])
    if name == "GaussLik":                 # gaussian.jl:26-28
        s = math.exp(lik[1])
        return (-0.5 * math.log(2 * math.pi) - math.log(s)) - 0.5 * ((np.asarray(y) - f) / s) ** 2
    if name == "PoisLik":                  # poisson.jl:13-16
        y = np.asarray(y)
        return y * f - np.exp(f) - gammaln(1.0 + y)
    if name == "StuTLik":                  # studentT.jl:29-34
        nu, s = lik[1], math.exp(lik[2])
        c = gammaln(0.5 * (nu + 1)) - gammaln(0.5 * nu) - 0.5 * math.log(math.pi * nu) - math.log(s)
        return np.array([c - (0.5 * (nu + 1)) * math.log(1 + (1 / nu) * ((yi - fi) / s) ** 2) for fi, yi in zip(f, y)])
    raise ValueError(lik)


def dlog_dens_df(lik, f, y):
    name = lik[0]
    if name == "BernLik":                  # bernoulli.jl:16-18
        return np.array([_phi(fi) / _Phi(fi) if yi else -_phi(fi) / (1.0 - _Phi(fi)) for fi, yi in zip(f, y)])
    if name == "BinLik":                   # binomial.jl:21-23
        n = lik[1]
        return np.array([yi / (1.0 + math.exp(fi)) - (n - yi) * math.exp(fi) / (1 + math.exp(fi)) for fi, yi in zip(f, y)])
    if name == "ExpLik":                   # exponential.jl:19-21
        return np.array([yi * math.exp(-fi) - 1 for fi, yi in zip(f, y)])
    if name == "GaussLik":                 # gaussian.jl:31-33
        s = math.exp(lik[1])
        return np.array([(yi - fi) / s ** 2 for fi, yi in zip(f, y)])
    if name == "PoisLik":                  # poisson.jl:19-21
        return np.asarray(y) - np.exp(f)
    if name == "StuTLik":                  # studentT.jl:37-41
        nu, s = lik[1], math.exp(lik[2])
        return np.array([(nu + 1) * (yi - fi) / (nu * s ** 2 + (yi - fi) ** 2) for fi, yi in zip(f, y)])
    raise ValueError(lik)


def dlog_dens_dθ(lik, f, y):
    """N x num_params(lik)"""
    name = lik[0]
    if name == "GaussLik":                 # gaussian.jl:36-38
        s = math.exp(lik[1])
        return s * np.array([[-1 / s + 1 / s ** 3 * (yi - fi) ** 2] for fi, yi in zip(f, y)])
    if name == "StuTLik":                  # studentT.jl:44-48
        nu, s = lik[1], math.exp(lik[2])
        return s * np.array([[-1 / s + (nu + 1) * (yi - fi) ** 2 / (nu * s ** 3 + s * (yi - fi) ** 2)] for fi, yi in zip(f, y)])
    return np.zeros((len(f), 0))


def lik_num_params(lik):
    return 1 if lik[0] in ("GaussLik", "StuTLik") else 0


def mean_lik(lik, f):
    name = lik[0]
    if name == "BernLik":                  # bernoulli.jl:21
        return np.array([_Phi(fi) for fi in f])
    if name == "BinLik":                   # binomial.jl:26
        return np.array([lik[1] * math.exp(fi) / (1.0 + math.exp(fi)) for fi in f])
    if name in ("ExpLik", "PoisLik"):      # exponential.jl:24, poisson.jl:24
        return np.exp(f)
    if name in ("GaussLik", "StuTLik"):    # gaussian.jl:41, studentT.jl:51
        return np.asarray(f, dtype=np.float64)
    raise ValueError(lik)


def var_lik(lik, f):
    name = lik[0]
    if name == "BernLik":                  # bernoulli.jl:22
        return np.array([_Phi(fi) * (1 - _Phi(fi)) for fi in f])
    if name == "BinLik":                   # binomial.jl:27
        return np.array([lik[1] * (math.exp(fi) / (1.0 + math.exp(fi))) * (1.0 / (1.0 + math.exp(fi))) for fi in f])
    if name == "ExpLik":                   # exponential.jl:25
        return np.exp(f) ** 2
    if name == "PoisLik":                  # poisson.jl:25
        return np.exp(f)
    if name == "GaussLik":                 # gaussian.jl:42
        return np.ones(len(f)) * math.exp(lik[1]) ** 2
    if name == "StuTLik":                  # studentT.jl:52
        nu = lik[1]
        return math.exp(lik[2]) ** 2 * (nu / (nu - 2.0)) * np.ones(len(f))
    raise ValueError(lik)


def predict_obs_quadrature(lik, fmean, fvar):
    """likelihoods.jl:16-31"""
    nodes, weights = np.polynomial.hermite.hermgauss(20)
    weights = weights / math.sqrt(math.pi)
    f = np.asarray(fmean)[:, None] + np.sqrt(2 * np.asarray(fvar))[:, None] * nodes[None, :]
    mL = np.empty(f.shape); vL = np.empty(f.shape)
    for i in range(nodes.size):
        mL[:, i] = mean_lik(lik, f[:, i])
        vL[:, i] = var_lik(lik, f[:, i])
    mu = mL @ weights
    return mu, (vL + mL ** 2) @ weights - mu ** 2


def predict_obs(lik, fmean, fvar):
    if lik[0] == "BernLik":                # bernoulli.jl:29-32
        p = np.array([_Phi(fm / math.sqrt(1 + fv)) for fm, fv in zip(fmean, fvar)])
        return p, p - p * p
    if lik[0] == "GaussLik":               # gaussian.jl:55-57
        return np.asarray(fmean), np.asarray(fvar) + math.exp(lik[1]) ** 2
    return predict_obs_quadrature(lik, fmean, fvar)


# ---- reverse-mode Cholesky -------------------------------------------------------------------------------------------
def chol_unblocked_rev(L, A_bar):
    """chol_unblocked_rev!(L, A_bar) (chol_utils.jl:15-39), in place on A_bar (0-based port of level2partition)."""
    N = A_bar.shape[0]
    for j in range(N - 1, -1, -1):
        r, d, B, c = L[j, :j], L[j, j], L[j + 1:, :j], L[j + 1:, j]
        A_bar[j, j] -= A_bar[j + 1:, j] @ c / d                     # d_bar -= dot(c_bar, c) / d
        A_bar[j, j] /= d
        A_bar[j + 1:, j] /= d                                       # c_bar ./= d
        A_bar[j, :j] -= A_bar[j, j] * r                             # r_bar -= d_bar r
        A_bar[j, :j] -= B.T @ A_bar[j + 1:, j]                      # gemv!('T', -1, B, c_bar, 1, r_bar)
        A_bar[j + 1:, :j] -= np.outer(A_bar[j + 1:, j], r)          # ger!(-1, c_bar, r, B_bar)
        A_bar[j, j] /= 2
    return A_bar


def L_bar_literal(L, g, v):
    """get_L_bar! + the diagonal doubling of dll_kern! (GPA.jl:130-143, 165-170)"""
    Lb = np.tril(np.outer(g, v))
    chol_unblocked_rev(np.tril(L), Lb)
    Lb[np.diag_indices_from(Lb)] *= 2
    return Lb


def dmll_kern_contract(A, grads):
    """dmll_kern! (GPE.jl:219-241) with ααinvcKI = A: sum_j A_jj dK_jj / 2 + sum_{i>j} A_ij dK_ij"""
    return np.array([0.5 * np.sum(np.diag(A) * np.diag(G)) + np.sum(np.tril(A, -1) * G) for G in grads])


def S_closed(L, g, v):
    """S = W' M_s W, W = L^-1, M_s[i,j] = u[max(i,j)] v[min(i,j)], u = L' g (dense)"""
    n = L.shape[0]
    W = sl.solve_triangular(L, np.eye(n), lower=True)
    u = L.T @ g
    I, J = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    Ms = np.where(I >= J, u[I] * v[J], u[J] * v[I])
    return W.T @ Ms @ W


def S_lower_scans(L, g, v):
    """the device's route: Z[i,b] = u_i sum_{b<=j<=i} v_j W[j,b] + v_i sum_{j>i} u_j W[j,b] (a prefix and a suffix scan down
    each column of W), then S[a,b] = sum_{i>=a} W[i,a] Z[i,b] for a >= b.  Returns the lower triangle of S."""
    n = L.shape[0]
    W = sl.solve_triangular(L, np.eye(n), lower=True)
    u = L.T @ g
    Z = np.zeros((n, n))
    for b in range(n):
        w = W[b:, b]
        pre = np.cumsum(v[b:] * w)                                  # inclusive prefix of v w
        uw = u[b:] * w
        suf = np.concatenate([np.cumsum(uw[::-1])[::-1][1:], [0.0]])   # exclusive suffix of u w
        Z[b:, b] = u[b:] * pre + v[b:] * suf
    S = np.zeros((n, n))
    for a in range(n):
        S[a, :a + 1] = W[a:, a] @ Z[a:, :a + 1]
    return S


# ---- GPA --------------------------------------------------------------------------------------------------------------
def update_target(spec, X, y, mspec, lik, v, init=False):
    """update_target!(gp::GPA) (GPA.jl:261-266 via update_ll! :118-128 and update_cK! :111-114, logNoise = -20);
    init=True: initialise_target! (:245-250, cK = PDMat(Σ + 1e-6 I), :101-109)."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    n = X.shape[0]
    K = cov(spec, X) + (1e-6 if init else math.exp(2 * -20.0)) * np.eye(n)
    L = np.linalg.cholesky(K)
    mu, MG = mean_and_grads(mspec, X)
    f = L @ v + mu                                                  # unwhiten(gp.cK, gp.v) + gp.μ
    ll = float(np.sum(log_dens(lik, f, y)))
    target = ll - (v @ v + LOG2PI * n) / 2
    return dict(L=L, K=K, mu=mu, MG=MG, f=f, ll=ll, target=target)


def update_dll(spec, X, y, mspec, lik, v, method="literal"):
    """update_dll! (GPA.jl:183-228) + update_dtarget! (:268-272, prior -v).  Order [v; lik; mean; kernel]."""
    o = update_target(spec, X, y, mspec, lik, v)
    L, f = o["L"], o["f"]
    g = dlog_dens_df(lik, f, y)                                    # precompute! (:158-163)
    u = L.T @ g                                                     # mul!(.., gp.cK.chol.U, dl_df)  (:200)
    dlik = np.sum(dlog_dens_dθ(lik, f, y), axis=0)                  # (:203-209)
    dmean = o["MG"].T @ g                                           # dmll_mean!(dll, mean, x, dl_df) (:174-176)
    _, grads = cov_and_grads(spec, X, None, True)
    if method == "literal":
        dk = dmll_kern_contract(L_bar_literal(L, g, v), grads)      # dll_kern! (:164-173)
    else:
        S = S_closed(L, g, v)
        dk = np.array([0.5 * np.sum(S * G) for G in grads])
    dll = np.concatenate([u, dlik, dmean, dk])
    dtarget = dll.copy()
    dtarget[:v.size] -= v
    o.update(g=g, u=u, dlik=dlik, dmean=dmean, dk=dk, dll=dll, dtarget=dtarget)
    return o


def predict_f(spec, X, mspec, o, Xs, full_cov=False):
    """predict_f(gp::GPA, x) (GPA.jl:294 -> predictMVN, GP.jl:25-79): alpha = cK \\ unwhiten(cK, v)"""
    L = o["L"]
    alpha = sl.cho_solve((L, True), o["f"] - o["mu"])
    Kc = cov(spec, X, Xs)
    mx, _ = mean_and_grads(mspec, Xs)
    mu = mx + Kc.T @ alpha
    V = sl.solve_triangular(L, Kc, lower=True)
    Kp = cov(spec, Xs)
    if full_cov:
        return mu, Kp - V.T @ V
    return mu, np.maximum(np.diag(Kp) - np.sum(V * V, axis=0), 0.0)


def predict_y(spec, X, mspec, lik, o, Xs):
    """predict_y(gp::GPA, x) (GPA.jl:303-306)"""
    mu, s2 = predict_f(spec, X, mspec, o, Xs)
    return predict_obs(lik, mu, s2)
