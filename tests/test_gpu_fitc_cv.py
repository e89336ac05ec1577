"""GPU: cross-validation on the sparse engine (gpb200_fitc_get_inverse_diag / _cv_param / _cv_block) for FITC, DTC and SoR,
against the dense restatement of tests/fitc_cv_oracle.py (Sigma and dSigma_j formed densely, the oracle's literal
cross-validation bodies on top).  Bounds scale with the measured cond(K_uu) cond(Sigma) eps: the device works through the
two M x M inverses, the oracle through a dense N x N solve, and the two orders differ by about that much."""
import numpy as np
import pytest

import fitc_cv_oracle as fco
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _kernel(kname):
    import gpb200 as g
    return g.SEIso(-0.6, 0.1) if kname == "SEIso" else g.Mat32Iso(-0.4, -0.1) + g.Noise(-1.3)


def _problem(N, M, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-2.0, 2.0, (M, d))                     # not training points: the Noise kernel stays off K_fu
    return X, y, Xu


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _oracle_mode(strategy):
    return "FITC" if strategy == "FITC" else "SoR"         # DTC trains with SoR's covariance


@pytest.mark.parametrize("N,M", [(300, 64), (300, 256), (3000, 64), (3000, 256)])
@pytest.mark.parametrize("kname", ["SEIso", "Mat32+Noise"])
@pytest.mark.parametrize("strategy", ["FITC", "DTC", "SoR"])
def test_sparse_cv_matches_dense_restatement(strategy, kname, N, M):
    import gpb200 as g
    d = 3
    X, y, Xu = _problem(N, M, d, N + M)
    k = _kernel(kname)
    ln = -1.0
    gp = getattr(g, strategy)(X.T, Xu.T, y, g.MeanZero(), k, ln)
    spec = k.spec()
    Sigma, grads = fco.sigma_and_grads(spec, X, Xu, ln, _oracle_mode(strategy))
    w = np.linalg.eigvalsh(orc.cov(spec, Xu) + 1e-10 * np.eye(M))
    ws = np.linalg.eigvalsh(Sigma)
    cond_u, cond_s = float(w[-1] / w[0]), float(ws[-1] / ws[0])
    tol = max(1e-9, 64.0 * cond_u * cond_s * EPS)
    alpha = np.linalg.solve(Sigma, y)
    assert _rel(gp.alpha, alpha) <= tol
    f = fco.cv_dict(Sigma, gp.alpha)
    folds = np.array_split(np.random.default_rng(1).permutation(N), 6 if N > 1000 else 10)
    e = {}
    mu, s2 = gp.predict_LOO()
    mo, so = orc.predict_loo(f, y)
    e["predict_LOO"] = max(_rel(mu, mo), _rel(s2, so))
    e["logp_LOO"] = _rel(gp.logp_LOO(), orc.logp_loo(f, y))
    e["dlogp_LOO"] = _rel(gp.dlogp_LOO(), fco.dlogp_loo(Sigma, grads, gp.alpha, y, ln))
    mus, Ss = gp.predict_CVfold(folds)
    mos, Sos = orc.predict_cvfold(f, y, folds)
    e["predict_CVfold"] = max(max(_rel(a, b) for a, b in zip(mus, mos)), max(_rel(a, b) for a, b in zip(Ss, Sos)))
    e["logp_CVfold"] = _rel(gp.logp_CVfold(folds), orc.logp_cvfold(f, y, folds))
    e["dlogp_CVfold"] = _rel(gp.dlogp_CVfold(folds), fco.dlogp_cvfold(Sigma, grads, gp.alpha, y, ln, folds))
    print("%s %s N=%d M=%d cond(K_uu)=%.1e cond(Sigma)=%.1e bound %.1e: %s"
          % (strategy, kname, N, M, cond_u, cond_s, tol, " ".join("%s %.1e" % kv for kv in e.items())))
    assert all(v <= tol for v in e.values()), e


@pytest.mark.parametrize("strategy", ["FITC", "SoR"])
def test_cv_gradients_vs_finite_differences(strategy):
    """central differences of the device logp_LOO / logp_CVfold against the device gradients [noise; kernel]"""
    import gpb200 as g
    N, M, d = 800, 60, 2
    X, y, Xu = _problem(N, M, d, 5)
    k = g.SEIso(-0.5, 0.0) + g.Noise(-1.5)
    gp = getattr(g, strategy)(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    folds = np.array_split(np.random.default_rng(2).permutation(N), 8)
    gl, gf = gp.dlogp_LOO(), gp.dlogp_CVfold(folds)
    p0 = [gp.logNoise] + list(k.get_params())
    h = 1e-5
    for i in range(len(p0)):
        v = []
        for sgn in (+1, -1):
            p = list(p0); p[i] += sgn * h
            gp.logNoise = p[0]; k.set_params(p[1:]); gp.update_mll()
            v.append((gp.logp_LOO(), gp.logp_CVfold(folds)))
        fl, ff = (v[0][0] - v[1][0]) / (2 * h), (v[0][1] - v[1][1]) / (2 * h)
        print("%s param %d: LOO fd %.8e dev %.8e | fold fd %.8e dev %.8e" % (strategy, i, fl, gl[i], ff, gf[i]))
        assert abs(fl - gl[i]) <= 1e-5 * max(abs(fl), 1.0), (i, fl, gl[i])
        assert abs(ff - gf[i]) <= 1e-5 * max(abs(ff), 1.0), (i, ff, gf[i])
    gp.logNoise = p0[0]; k.set_params(p0[1:]); gp.update_mll()


def _state(gp, Xs):
    eng = gp._eng
    _, mll, logdet = eng.mll(gp.y)
    return [np.array([mll, logdet, eng.grad_noise()]), eng.grad_kernel(), *eng.predict(Xs), eng.predict_cov(Xs[:50])[1]]


@pytest.mark.parametrize("strategy", ["FITC", "DTC", "SoR"])
def test_bitwise_repeat_and_untouched_state(strategy):
    """two calls return bitwise equal results; after CV calls the likelihood, gradients and predictions of the handle are
    bitwise those of a fresh handle"""
    import gpb200 as g
    N, M, d = 2500, 130, 3
    X, y, Xu = _problem(N, M, d, 9)
    Xs = np.random.default_rng(3).standard_normal((200, d))
    k = g.Mat32Iso(-0.4, -0.1) + g.Noise(-1.3)
    gp = getattr(g, strategy)(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    eng = gp._eng
    V = np.arange(3, N, 11)
    a = [eng.inverse_diag(), *eng.cv_param(1), eng.cv_block(1, V), eng.cv_block(0, V), *eng.cv_param(-1), eng.cv_block(1, V)]
    b = [eng.inverse_diag(), *eng.cv_param(1), eng.cv_block(1, V), eng.cv_block(0, V), *eng.cv_param(-1), eng.cv_block(1, V)]
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    after = _state(gp, Xs)
    fresh = getattr(g, strategy)(X.T, Xu.T, y, g.MeanZero(), _kernel("Mat32+Noise"), -1.0)
    ref = _state(fresh, Xs)
    assert all(np.array_equal(u, v) for u, v in zip(after, ref))


def test_error_codes():
    import gpb200 as g
    from gpb200 import capi
    N, M, d = 400, 40, 2
    X, y, Xu = _problem(N, M, d, 4)
    k = g.SEIso(-0.5, 0.0)
    eng = capi.FitcEngine(0)
    eng.set_data(X, Xu)
    ops, dims, theta, _ = g.kernels.flatten(k, d)
    eng.set_kernel(ops, dims, theta.size)
    lib, h = eng._lib, eng._h
    out = np.empty(N); out2 = np.empty(N); blk = np.empty(16)
    idx = np.arange(4, dtype=np.int64)
    ip = idx.ctypes.data_as(capi.C.POINTER(capi.C.c_int64))
    dp = capi._as_dp
    assert lib.gpb200_fitc_get_inverse_diag(h, dp(out)) == capi.ESTATE
    eng.factorize(theta, -1.0)
    assert lib.gpb200_fitc_cv_param(h, 0, None, dp(out), dp(out2)) == capi.ESTATE     # factorize without mll
    eng.mll(y)
    assert lib.gpb200_fitc_cv_block(h, 1, 4, ip, dp(blk)) == capi.ESTATE               # which = 1 before any cv_param
    assert lib.gpb200_fitc_cv_param(h, theta.size, None, dp(out), dp(out2)) == capi.EINVAL
    assert lib.gpb200_fitc_cv_param(h, -2, None, dp(out), dp(out2)) == capi.EINVAL
    assert lib.gpb200_fitc_cv_param(h, 0, None, dp(out), dp(out2)) == capi.OK
    assert lib.gpb200_fitc_cv_block(h, 1, 4, ip, dp(blk)) == capi.OK
    assert lib.gpb200_fitc_cv_block(h, 2, 4, ip, dp(blk)) == capi.EINVAL
    bad = np.array([0, N], dtype=np.int64)
    assert lib.gpb200_fitc_cv_block(h, 0, 2, bad.ctypes.data_as(capi.C.POINTER(capi.C.c_int64)), dp(blk)) == capi.EINVAL
    eng.factorize(theta, -1.0); eng.mll(y)
    assert lib.gpb200_fitc_cv_block(h, 1, 4, ip, dp(blk)) == capi.ESTATE               # the last factorize cleared M_j
    # FSA (mode 3): EINVAL from the engine, ValueError from the host class
    blocks = [np.arange(i, min(i + 100, N)) for i in range(0, N, 100)]
    fsa = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.SEIso(-0.5, 0.0), -1.0)
    assert fsa._eng._lib.gpb200_fitc_get_inverse_diag(fsa._eng._h, dp(out)) == capi.EINVAL
    assert "FSA" in fsa._eng._lib.gpb200_fitc_last_error(fsa._eng._h).decode()
    for call in (fsa.predict_LOO, fsa.logp_LOO, fsa.dlogp_LOO, lambda: fsa.predict_CVfold([idx]), lambda: fsa.dlogp_CVfold([idx])):
        with pytest.raises(ValueError):
            call()
    # mean parameters: NotImplementedError as in the reference (crossvalidation.jl:168, 330)
    gm = g.FITC(X.T, Xu.T, y, g.MeanConst(0.2), g.SEIso(-0.5, 0.0), -1.0)
    with pytest.raises(NotImplementedError):
        gm.dlogp_LOO(domean=True)
    with pytest.raises(NotImplementedError):
        gm.dlogp_CVfold([idx], domean=True)
    eng.close()


@pytest.mark.slow
def test_full_size_fitc_cv():
    """N = 10^6, M = 4096, d = 8, SEIso: [Sigma^-1]_ii and a fold block on sampled rows against Sigma^-1 e_i from the engine's
    own mll solve (rhs e_i), and one directional finite difference of logp_LOO"""
    import gpb200 as g
    rng = np.random.default_rng(12)
    N, M, d = 1_000_000, 4096, 8
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1) / 2) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    k = g.SEIso(0.3, 0.0)
    gp = g.FITC(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    eng = gp._eng
    dg = eng.inverse_diag()
    rows = rng.choice(N, 4, replace=False)
    blk = eng.cv_block(0, rows)
    cols = []
    for i in rows:
        e = np.zeros(N); e[i] = 1.0
        cols.append(eng.mll(e)[0])
    ref = np.array([[c[j] for j in rows] for c in cols])
    print("full size: diag %s vs %s" % (dg[rows], np.diag(ref)))
    assert _rel(dg[rows], np.diag(ref)) <= 1e-6
    assert _rel(blk, ref) <= 1e-6
    gp.update_mll()
    grad = gp.dlogp_LOO()
    dirn = rng.standard_normal(grad.size); dirn /= np.linalg.norm(dirn)
    p0 = np.array([gp.logNoise] + list(k.get_params()))
    h = 1e-4
    v = []
    for sgn in (+1, -1):
        p = p0 + sgn * h * dirn
        gp.logNoise = p[0]; k.set_params(list(p[1:])); gp.update_mll()
        v.append(gp.logp_LOO())
    fd = (v[0] - v[1]) / (2 * h)
    print("full size: directional fd %.8e vs gradient %.8e" % (fd, grad @ dirn))
    assert abs(fd - grad @ dirn) <= 1e-4 * max(abs(fd), 1.0)
