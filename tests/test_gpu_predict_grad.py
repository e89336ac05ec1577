"""GPU: predictive gradients with respect to the test inputs (gpb200_predict_grad, GPE / ElasticGPE / GPA.predict_f_grad)
against the numpy restatement in xgrad_oracle, against predict_f itself (bitwise), across chunkings, against central
differences of the device predict_f at N = 32768, and the state the call must leave alone."""
import functools

import numpy as np
import pytest

from conftest import kernel_zoo, make_data
from oracle import gp_oracle as orc
import xgrad_oracle as xo

pytestmark = pytest.mark.gpu

LOGNOISE = -1.0


def _mean(d):
    import gpb200 as g
    return g.MeanLin([0.3 * (p + 1) for p in range(d)])


@functools.lru_cache(maxsize=None)
def _fit(name, N):
    import gpb200 as g
    kern = dict(kernel_zoo(3))[name]
    X, y, _ = make_data(N, 3, 11)
    gp = g.GPE(X.T, y, _mean(3), kern, LOGNOISE)
    f = orc.fit(kern.spec(), X, y, LOGNOISE, _mean(3).spec())
    return gp, kern.spec(), X, f


def _rel(got, want):
    return np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-300)


@pytest.mark.parametrize("N", [700, 3000])
@pytest.mark.parametrize("name", [n for n, _ in kernel_zoo(3)])
def test_zoo_parity(name, N):
    gp, spec, X, f = _fit(name, N)
    for M in (1, 130):
        Xs = 0.8 * np.random.default_rng(M + N).standard_normal((M, 3))
        mu, s2, dmu, ds2 = gp.predict_f_grad(Xs.T)
        wmu, wvar, wdmu, wdvar = xo.predict_f_grad(spec, X, f, Xs, _mean(3).spec())
        assert dmu.shape == (3, M) and ds2.shape == (3, M)
        assert _rel(mu, wmu) <= 1e-10
        assert _rel(dmu.T, wdmu) <= 1e-8, (name, N, M, _rel(dmu.T, wdmu))
        keep = wvar > 0.0
        assert _rel(ds2.T[keep], wdvar[keep]) <= 1e-8, (name, N, M, _rel(ds2.T[keep], wdvar[keep]))


@pytest.mark.parametrize("name", ["SE+RQ", "Mat12Iso", "Mat12Ard", "(SE+Mat12)*RQ", "Periodic(1d)", "MaunaLoa-like"])
def test_on_training_points(name):
    """a test point equal to a training input: the r = 0 rules (the limit, Mat12's 0, Periodic's guarded sin(2u)/r) give
    finite gradients that match the oracle's"""
    gp, spec, X, f = _fit(name, 700)
    Xs = np.vstack([X[[5, 77, 300]], 0.5 * X[[1, 2]]])
    _, _, dmu, ds2 = gp.predict_f_grad(Xs.T)
    _, _, wdmu, wdvar = xo.predict_f_grad(spec, X, f, Xs, _mean(3).spec())
    assert np.all(np.isfinite(dmu)) and np.all(np.isfinite(ds2))
    assert _rel(dmu.T, wdmu) <= 1e-8 and _rel(ds2.T, wdvar) <= 1e-8


@pytest.mark.parametrize("name", ["SEIso", "(SE+Mat12)*RQ", "LinIso+Const"])
def test_agrees_with_predict_bitwise(name):
    gp, _, _, _ = _fit(name, 3000)
    Xs = np.random.default_rng(3).standard_normal((300, 3))
    e = gp._eng
    mu0, var0, _ = e.predict(Xs, None)
    mu1, var1, _, _ = e.predict_grad(Xs)
    mu2, var2, dmu2, dvar2 = e.predict_grad(Xs, want_var=False)
    assert np.array_equal(mu0, mu1) and np.array_equal(var0, var1) and np.array_equal(mu0, mu2)
    assert var2 is None and dvar2 is None
    mu, s2 = gp.predict_f(Xs.T)
    mug, s2g, _, _ = gp.predict_f_grad(Xs.T)
    assert np.array_equal(mu, mug) and np.array_equal(s2, s2g)


@pytest.mark.parametrize("name", ["SEIso", "MaunaLoa-like"])
def test_chunked_and_repeated_bitwise(name, monkeypatch):
    gp, _, _, _ = _fit(name, 3000)
    Xs = np.random.default_rng(4).standard_normal((300, 3))
    e = gp._eng
    a = e.predict_grad(Xs)
    b = e.predict_grad(Xs)
    monkeypatch.setenv("GPB200_PREDICT_CHUNK", "128")
    c = e.predict_grad(Xs)
    dmu_only = e.predict_grad(Xs, want_var=False)
    for u, v, w in zip(a, b, c):
        assert np.array_equal(u, v) and np.array_equal(u, w)
    assert np.array_equal(dmu_only[2], a[2])


def _engine_pair(X, kern):
    import gpb200 as g
    from gpb200.kernels import flatten
    ops, dims, theta, _ = flatten(kern, X.shape[1])
    es = []
    for _ in range(2):
        e = g.Engine(0)
        e.set_data(X)
        e.set_kernel(ops, dims, theta.size)
        e.factorize(theta, LOGNOISE)
        es.append(e)
    return es


def test_state_unchanged():
    """grad_kernel, cv_param, cv_block, mll, solve and gpa_grad are bitwise the same with and without a predict_grad in between;
    predict_grad fills F's strict-upper tiles with L', which the inverse merges and GPA's scans overwrite before reading"""
    import gpb200 as g
    X, y, _ = make_data(1000, 3, 21)
    kern = g.SEIso(0.2, 0.1) * g.RQIso(0.3, 0.0, 0.2)
    a, b = _engine_pair(X, kern)
    Xs = np.random.default_rng(5).standard_normal((200, 3))
    r = np.random.default_rng(6).standard_normal(1000)
    V = np.arange(0, 1000, 7)

    def run(e, pg):
        out = []
        if pg:
            e.predict_grad(Xs, alpha=r)
        out.append(e.mll(y))
        if pg:
            e.predict_grad(Xs)
        e.grad_prepare()
        out.append(e.grad_kernel())
        if pg:
            e.predict_grad(Xs)
        out.append(e.cv_param(0))
        out.append(e.cv_block(0, V))
        out.append(e.cv_param(-1))
        if pg:
            e.predict_grad(Xs)
        out.append(e.cv_block(1, V))
        out.append(e.grad_kernel())
        out.append(e.solve(r))
        if pg:
            e.predict_grad(Xs)
        out.append(e.gpa_grad(r, y))
        if pg:
            e.predict_grad(Xs, alpha=r)
        out.append(e.gpa_grad(y, r))
        e.mll(y)
        e.grad_prepare()
        out.append(e.grad_kernel())
        return out

    ra, rb = run(a, True), run(b, False)
    for u, v in zip(ra, rb):
        for p, q in zip(u, v):
            assert np.array_equal(np.asarray(p), np.asarray(q))
    a.close(); b.close()


@pytest.mark.parametrize("k", [1, 200])
def test_elastic_append(k):
    import gpb200 as g
    X, y, _ = make_data(1500 + k, 3, 31)
    kern = g.Mat52Iso(0.3, 0.1)
    el = g.ElasticGPE(X[:1500].T, y[:1500], _mean(3), kern, LOGNOISE, capacity=2000)
    el.append(X[1500:].T, y[1500:])
    fresh = g.GPE(X.T, y, _mean(3), g.Mat52Iso(0.3, 0.1), LOGNOISE)
    Xs = np.random.default_rng(7).standard_normal((150, 3))
    a, b = el.predict_f_grad(Xs.T), fresh.predict_f_grad(Xs.T)
    for u, v in zip(a, b):
        assert _rel(u, v) <= 1e-9


@pytest.mark.parametrize("lname", ["BernLik", "PoisLik"])
def test_gpa(lname):
    import scipy.linalg as sl
    from test_gpu_gpa import _gpa
    gp, X, y, _ = _gpa(lname, "SE_Noise", 500)
    gp.update_target()
    Xs = 2 * np.pi * np.random.default_rng(8).random((40, 3))
    mu, s2, dmu, ds2 = gp.predict_f_grad(Xs.T)
    K = orc.cov(gp.kernel.spec(), X) + np.exp(2 * -20.0) * np.eye(X.shape[0])
    L = np.linalg.cholesky(K)
    alpha = sl.cho_solve((L, True), L @ gp.v)
    wmu, wvar, wdmu, wdvar = xo.predict_f_grad(gp.kernel.spec(), X, dict(U=L.T), Xs, gp.mean.spec(), alpha=alpha)
    pm, ps2 = gp.predict_f(Xs.T)
    assert np.array_equal(mu, pm) and np.array_equal(s2, ps2)
    assert _rel(dmu.T, wdmu) <= 1e-7, _rel(dmu.T, wdmu)
    keep = wvar > 0.0
    assert _rel(ds2.T[keep], wdvar[keep]) <= 1e-7, _rel(ds2.T[keep], wdvar[keep])


@pytest.mark.parametrize("case", ["SEIso d=8", "Mat32Iso+RQIso"])
def test_large_n_directional_differences(case):
    """N = 32768: central differences of the device predict_f along a random direction per test point, 64 points"""
    import gpb200 as g
    d = 8 if case.startswith("SEIso") else 3
    X, y, _ = make_data(32768, d, 41)
    kern = g.SEIso(0.5, 0.0) if d == 8 else g.Mat32Iso(0.2, 0.0) + g.RQIso(0.4, -0.3, 0.1)
    gp = g.GPE(X.T, y, _mean(d), kern, -1.5)
    rng = np.random.default_rng(9)
    Xs = rng.standard_normal((64, d))
    Dv = rng.standard_normal((64, d))
    Dv /= np.linalg.norm(Dv, axis=1, keepdims=True)
    _, _, dmu, ds2 = gp.predict_f_grad(Xs.T)
    h = 1e-4
    mp, vp = gp.predict_f((Xs + h * Dv).T)
    mm, vm = gp.predict_f((Xs - h * Dv).T)
    fd_mu, fd_var = (mp - mm) / (2 * h), (vp - vm) / (2 * h)
    g_mu, g_var = np.sum(dmu.T * Dv, axis=1), np.sum(ds2.T * Dv, axis=1)
    assert _rel(g_mu, fd_mu) <= 1e-6, _rel(g_mu, fd_mu)
    assert _rel(g_var, fd_var) <= 1e-6, _rel(g_var, fd_var)


def test_error_codes():
    import gpb200 as g
    from gpb200 import capi
    from gpb200.kernels import flatten
    X, y, _ = make_data(300, 3, 61)
    kern = g.SEIso(0.2, 0.1)
    e = g.Engine(0)
    e.set_data(X)
    ops, dims, theta, _ = flatten(kern, 3)
    e.set_kernel(ops, dims, theta.size)
    xs = np.zeros((4, 3))
    with pytest.raises(ValueError, match="factorize first"):
        e.predict_grad(xs, alpha=np.zeros(300))
    e.factorize(theta, LOGNOISE)
    with pytest.raises(ValueError, match="no alpha"):
        e.predict_grad(xs)
    lib, h, dp = e._lib, e._h, capi._as_dp
    mu, var, dmu, dvar, a = np.empty(4), np.empty(4), np.empty((4, 3)), np.empty((4, 3)), np.zeros(300)
    assert lib.gpb200_predict_grad(None, 4, dp(xs), 3, dp(a), dp(mu), dp(var), dp(dmu), dp(dvar)) == capi.EINVAL
    for args in [(0, dp(xs), 3, dp(a), dp(mu), dp(var), dp(dmu), dp(dvar)),
                 (4, None, 3, dp(a), dp(mu), dp(var), dp(dmu), dp(dvar)),
                 (4, dp(xs), 2, dp(a), dp(mu), dp(var), dp(dmu), dp(dvar)),
                 (4, dp(xs), 3, dp(a), None, dp(var), dp(dmu), dp(dvar)),
                 (4, dp(xs), 3, dp(a), dp(mu), dp(var), None, dp(dvar)),
                 (4, dp(xs), 3, dp(a), dp(mu), dp(var), dp(dmu), None),
                 (4, dp(xs), 3, dp(a), dp(mu), None, dp(dmu), dp(dvar))]:
        assert lib.gpb200_predict_grad(h, *args) == capi.EINVAL, args
    assert lib.gpb200_predict_grad(h, 4, dp(xs), 3, dp(a), dp(mu), None, dp(dmu), None) == capi.OK
    e.close()
    grp = g.LocalGroupEngine(2, rb=1)
    gs = g.GPE(X.T, y, g.MeanZero(), g.SEIso(0.2, 0.1), LOGNOISE, engine=grp)
    with pytest.raises(ValueError, match="single GPU"):
        gs.predict_f_grad(xs.T)
    grp.close()
