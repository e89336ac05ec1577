"""GPU: the BASELINE.json configurations that had no parity test at their own size.

C3  GPE Sum(SEArd, Periodic*SEArd, RQIso, SEArd) Mauna-Loa-style, N=16384, d=1 (SURVEY.md §8(d), kernel structure of
    docs/src/mauna_loa.md:21): the numpy oracle fits in RAM here (2 GB per matrix), so mll / alpha / predict_f are
    compared with it at the north-star tolerance 1e-10; the 13-parameter gradient (the oracle's literal dmll_kern! needs
    ~15 N x N temporaries) is checked by a directional finite difference of the already-verified mll plus the normwise
    backward residual of alpha that §8(d) prescribes.
C5  FITC SEIso N=1e6, M=8192 inducing, d=32 (test/test_sparse.jl:121-144 style, RNG-free properties): the residual
    Sigma alpha = r on sampled rows with Sigma = Lambda + K_fu K_uu^-1 K_uf rebuilt on the host cores (K_uf streamed),
    logdet via the matrix-determinant lemma on the host, and a directional finite difference of the FITC mll."""
import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def test_c3_composite_mauna_loa_at_full_size():
    import gpb200 as g
    N = 16384
    rng = np.random.default_rng(3)
    x = np.sort(rng.uniform(1958, 2004, N))
    y = 315 + 1.5 * (x - 1958) + 3 * np.sin(2 * np.pi * x) + 0.3 * rng.standard_normal(N)
    y = (y - y.mean()) / y.std()
    xs = rng.uniform(2004, 2024, 2048)
    k = g.SEArd([4.0], 0.0) + g.Periodic(0.0, 0.0, 0.0) * g.SEArd([4.0], 0.0) + g.RQIso(0.0, 0.0, -1.0) + g.SEArd([-2.0], -2.0)
    gp = g.GPE(x[None, :], y, g.MeanZero(), k, 0.0)
    gp.update_target_and_dtarget()
    assert gp.dmll.size == 1 + 12
    X = x[:, None]
    o = orc.fit(k.spec(), X, y, 0.0)
    e_mll = abs(gp.mll - o["mll"]) / abs(o["mll"])
    e_al = _rel(gp.alpha, o["alpha"])
    print("C3 N=%d: mll rel err %.2e, alpha rel err %.2e" % (N, e_mll, e_al))
    assert e_mll <= 1e-10 and e_al <= 1e-10
    # normwise backward residual |K_y alpha - r| / (|K_y| |alpha|)  (SURVEY §8(d), ill-conditioning-proof)
    Ky = orc.gram(k.spec(), X, 0.0)
    res = np.linalg.norm(Ky @ gp.alpha - y) / (np.linalg.norm(Ky, 2 if N <= 2048 else "fro") * np.linalg.norm(gp.alpha))
    assert res <= 1e-14, res
    del Ky
    mu, s2 = gp.predict_f(xs[None, :])
    mo, vo = orc.predict_f(k.spec(), X, o, xs[:, None])
    assert _rel(mu, mo) <= 1e-10
    assert np.max(np.abs(s2 - vo)) <= 1e-10 * np.max(np.abs(vo)) + 1e-13
    # gradient: directional derivative vs central difference of the (oracle-verified) device mll
    p0 = gp.get_params(); g0 = gp.dtarget.copy()
    dirv = np.random.default_rng(0).standard_normal(p0.size); dirv /= np.linalg.norm(dirv)
    h = 1e-5
    gp.set_params(p0 + h * dirv); gp.update_target(); tp = gp.target
    gp.set_params(p0 - h * dirv); gp.update_target(); tm = gp.target
    fd = (tp - tm) / (2 * h)
    assert abs(fd - g0 @ dirv) <= 1e-6 * max(abs(fd), np.linalg.norm(g0)), (fd, g0 @ dirv)
    gp.set_params(p0)


def _host_kuf_pass(X, Xu, l2, s2, alpha, rows, nthreads):
    """b = K_uf alpha streamed over row chunks on the host cores (SEIso); also returns K_fu[rows, :]."""
    N, M = X.shape[0], Xu.shape[0]
    un = np.sum(Xu * Xu, axis=1)
    step = 4096
    starts = list(range(0, N, step))

    def work(r0):
        xc = X[r0:r0 + step]
        G = xc @ Xu.T
        G *= -2.0
        G += np.sum(xc * xc, axis=1)[:, None]
        G += un[None, :]
        np.maximum(G, 0.0, out=G)
        G *= -0.5 / l2
        np.exp(G, out=G)
        G *= s2
        return G.T @ alpha[r0:r0 + step]

    with ThreadPoolExecutor(nthreads) as ex:
        parts = list(ex.map(work, starts))
    b = np.sum(parts, axis=0)
    Kr = s2 * np.exp(-0.5 / l2 * np.maximum(
        np.sum(X[rows] ** 2, 1)[:, None] + un[None, :] - 2.0 * X[rows] @ Xu.T, 0.0))
    # exact (direct-difference) distances for the sampled rows: the property check must not inherit the
    # cancellation of the |x|^2 + |u|^2 - 2 x.u form
    for a, i in enumerate(rows):
        d2 = np.sum((Xu - X[i]) ** 2, axis=1)
        Kr[a] = s2 * np.exp(-0.5 * d2 / l2)
    return b, Kr


@pytest.mark.slow
def test_c5_fitc_properties_at_full_size():
    import gpb200 as g
    N, M, d = 1_000_000, 8192, 32
    rng = np.random.default_rng(5)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(axis=1) / math.sqrt(d)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]].copy()
    ll, ls, ln = math.log(4.0), 0.0, math.log(0.1)
    mean_y = float(y.mean())
    k = g.SEIso(ll, ls)
    gp = g.FITC(X.T, Xu.T, y, g.MeanConst(mean_y), k, ln)
    gp.update_mll_and_dmll()
    assert np.isfinite(gp.mll) and gp.dmll.size == 1 + 1 + 2
    l2, s2, nv = math.exp(2 * ll), math.exp(2 * ls), math.exp(2 * ln)
    r = y - mean_y
    rows = rng.choice(N, 48, replace=False)
    nthreads = min(32, os.cpu_count() or 1)
    b, Kr = _host_kuf_pass(X, Xu, l2, s2, gp.alpha, rows, nthreads)
    # K_uu (+1e-10, fitc.jl:139-141), direct differences via the oracle
    Kuu = orc.cov(k.spec(), Xu) + 1e-10 * np.eye(M)
    Lu = np.linalg.cholesky(Kuu)
    v = np.linalg.solve(Lu.T, np.linalg.solve(Lu, b))                       # K_uu^-1 K_uf alpha
    W = np.linalg.solve(Lu, Kr.T)                                           # L_uu^-1 k_ui
    lam = nv + s2 - np.sum(W * W, axis=0)                                   # Lambda_i (fitc.jl:146-148)
    sig_alpha = lam * gp.alpha[rows] + Kr @ v
    err = np.max(np.abs(sig_alpha - r[rows])) / np.max(np.abs(r))
    # The reference's Woodbury form (fitc.jl:33-36: alpha = L^-1 (r - K_fu S^-1 K_uf L^-1 r)) inherits
    # cond(Sigma_QR) ~ lambda_max(K_uf L^-1 K_fu) / lambda_min(K_uu) ~ (M N kbar^2 / sigma^2) / 0.86 ~ 1e10 at C5, so the
    # residual of ANY implementation of those formulas sits near cond * eps ~ 1e-6 |r| (the numpy oracle shows 3e-10 at
    # N=2e4, M=512 and 5e-10 at N=6e4, M=1024, growing with M N).
    scond = (M * N * 0.135 ** 2 / nv) / 0.86
    print("C5 residual (Sigma alpha - r) on 48 rows: %.2e |r|   (cond(Sigma_QR) ~ %.1e, cond*eps = %.1e)"
          % (err, scond, scond * np.finfo(float).eps))
    assert err <= 4.0 * scond * np.finfo(float).eps, err
    # directional finite difference of the FITC mll (test/test_sparse.jl:134-144 at scale)
    g0 = gp.dmll.copy(); p0 = np.array([ln, mean_y, ll, ls])
    dirv = np.array([0.5, 0.0, -0.4, 0.3])
    h = 5e-4                                  # mll ~ -1.8e5 carries ~1e-10 relative rounding: a smaller step drowns in it
    vals = []
    for sgn in (+1, -1):
        p = p0 + sgn * h * dirv
        gp.logNoise = p[0]; k.set_params([p[2], p[3]]); gp.update_mll(); vals.append(gp.mll)
    fd = (vals[0] - vals[1]) / (2 * h)
    gp.logNoise = ln; k.set_params([ll, ls])
    print("C5 directional derivative: fd %.6f analytic %.6f" % (fd, g0 @ dirv))
    assert abs(fd - g0 @ dirv) <= 1e-4 * abs(fd) + 1e-2, (fd, g0 @ dirv)
    # predictions: prior variance bounds and the mean at sampled training points (K_xu u, u = Sigma_QR^-1 K_uf Lambda^-1 r)
    gp.update_mll()
    Xs = rng.standard_normal((4096, d))
    mu, s2p = gp.predict_f(Xs.T)
    assert np.all(np.isfinite(mu)) and np.all(s2p >= 0.0) and np.all(s2p <= s2 * (1 + 1e-9))
