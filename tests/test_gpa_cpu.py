"""CPU: the GPA oracle (tests/gpa_oracle.py) pinned the way the reference pins GPA (test/gpa.jl: dtarget == central finite
differences of target for all six likelihoods), the closed form the device computes (S = W' M_s W from two scans and one
triangular product) against the literal reverse-mode Cholesky, and the host assembly of gpb200.GPA over a numpy stub engine."""
import math
import os
import re

import numpy as np
import pytest

import gpa_oracle as go
from oracle.gp_oracle import cov, cov_and_grads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIKS = ["BernLik", "BinLik", "ExpLik", "GaussLik", "PoisLik", "StuTLik"]


def gpa_problem(n=20, d=3, seed=1):
    """test/gpa.jl:8-20: X = 2π U(0,1), f = sum(sin)/d and one y vector per likelihood"""
    rng = np.random.default_rng(seed)
    X = 2 * np.pi * rng.random((n, d))
    f = np.sin(X).sum(axis=1) / d
    ys = dict(BernLik=rng.random(n) < np.abs(f),
              BinLik=rng.binomial(n, np.exp(f) / (1 + np.exp(f))).astype(np.int64),
              ExpLik=rng.exponential(f ** 2),
              GaussLik=f.copy(),
              PoisLik=rng.poisson(np.exp(f)).astype(np.int64),
              StuTLik=f + rng.standard_t(3, n))
    liks = dict(BernLik=("BernLik",), BinLik=("BinLik", n), ExpLik=("ExpLik",), GaussLik=("GaussLik", -1.0), PoisLik=("PoisLik",),
                StuTLik=("StuTLik", 3, 0.1))
    return X, ys, liks, rng


def _with_lik_param(lik, p):
    return lik[:-1] + (p,) if go.lik_num_params(lik) else lik


@pytest.mark.parametrize("name", LIKS)
def test_oracle_dtarget_matches_finite_differences(name):
    X, ys, liks, rng = gpa_problem()
    y, lik = ys[name], liks[name]
    n = X.shape[0]
    nl = go.lik_num_params(lik)
    params = 0.5 * rng.standard_normal(n + nl + 2)                     # [v; lik; kernel]: SE(0, 0), MeanZero

    def unpack(p):
        return p[:n], _with_lik_param(lik, p[n]) if nl else lik, ("SEIso", list(p[n + nl:]))

    def target(p):
        v, lk, spec = unpack(p)
        return go.update_target(spec, X, y, ("MeanZero",), lk, v)["target"]

    v, lk, spec = unpack(params)
    exact = go.update_dll(spec, X, y, ("MeanZero",), lk, v)["dtarget"]
    h = 1e-6
    num = np.array([(target(params + h * e) - target(params - h * e)) / (2 * h) for e in np.eye(params.size)])
    assert np.allclose(num, exact, rtol=1e-5, atol=1e-6), np.max(np.abs(num - exact))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_closed_form_matches_the_literal_reverse_cholesky(seed):
    rng = np.random.default_rng(seed)
    n = 300
    A = rng.standard_normal((n, n))
    K = A @ A.T / n + (0.5 + seed) * np.eye(n)
    L = np.linalg.cholesky(K)
    v, g = rng.standard_normal(n), rng.standard_normal(n) * (1 + seed)
    S = go.S_closed(L, g, v)
    Sl = go.S_lower_scans(L, g, v)
    assert np.max(np.abs(Sl - np.tril(S))) <= 1e-13 * np.max(np.abs(S))
    Lb = go.L_bar_literal(L, g, v)
    for _ in range(3):
        D = rng.standard_normal((n, n)); D = D + D.T
        lit = go.dmll_kern_contract(Lb, [D])[0]
        closed = 0.5 * (2 * np.sum(np.tril(Sl, -1) * D) + np.sum(np.diag(Sl) * np.diag(D)))
        assert abs(lit - closed) <= 1e-13 * (np.sum(np.abs(Lb * D)) + abs(lit)), (lit, closed)


def test_oracle_literal_and_closed_kernel_gradients_agree():
    X, ys, liks, rng = gpa_problem(n=60)
    v = rng.standard_normal(60)
    spec = ("Sum", ("SEIso", [0.2, 0.1]), ("Noise", [-1.0]))
    a = go.update_dll(spec, X, ys["PoisLik"], ("MeanConst", 0.3), liks["PoisLik"], v, method="literal")
    b = go.update_dll(spec, X, ys["PoisLik"], ("MeanConst", 0.3), liks["PoisLik"], v, method="closed")
    assert np.allclose(a["dtarget"], b["dtarget"], rtol=1e-11, atol=1e-12)


# ---- host assembly over a stub engine ----------------------------------------------------------------------------------
class StubEngine:
    """numpy stand-in for capi.Engine: the GPA host class sees the same calls, the oracle does the arithmetic"""

    def __init__(self, kernel):
        self.kernel, self.calls = kernel, []

    def set_data(self, x_pm):
        self.X = np.array(x_pm); self.N, self.d = self.X.shape

    def set_kernel(self, ops, dims, n_theta):
        self.n_theta = n_theta

    def factorize(self, theta, log_noise, extra_nugget=0.0):
        self.calls.append(("factorize", float(log_noise), float(extra_nugget)))
        K = cov(self.kernel.spec(), self.X) + (math.exp(2 * log_noise) + extra_nugget) * np.eye(self.N)
        self.L = np.linalg.cholesky(K)

    def unwhiten(self, v):
        return self.L @ v

    def solve(self, rhs):
        return np.linalg.solve(self.L @ self.L.T, rhs)

    def gpa_grad(self, v, dl_df, process=True, kern=True):
        self.calls.append(("gpa_grad", process, kern))
        S = go.S_closed(self.L, dl_df, v)
        _, grads = cov_and_grads(self.kernel.spec(), self.X, None, True)
        return (self.L.T @ dl_df if process else None), (np.array([0.5 * np.sum(S * G) for G in grads]) if kern else None)

    def predict(self, xs, alpha=None, want_var=True, full_cov=False):
        Kc = cov(self.kernel.spec(), self.X, xs)
        V = np.linalg.solve(self.L, Kc)
        Kp = cov(self.kernel.spec(), xs)
        return Kc.T @ alpha, np.diag(Kp) - np.sum(V * V, axis=0), (Kp - V.T @ V if full_cov else None)


def _stub_gpa(name="GaussLik", mean=None, n=30):
    import gpb200 as g
    X, ys, _, rng = gpa_problem(n=n)
    lik = dict(BernLik=g.BernLik(), BinLik=g.BinLik(n), ExpLik=g.ExpLik(), GaussLik=g.GaussLik(-1.0), PoisLik=g.PoisLik(),
               StuTLik=g.StuTLik(3, 0.1))[name]
    k = g.SEIso(0.1, 0.2) + g.Noise(-1.0)
    gp = g.GPA(X.T, ys[name], mean or g.MeanConst(0.2), k, lik, engine=StubEngine(k))
    return gp, X, ys[name], rng


def test_gp_with_a_likelihood_is_a_gpa_and_initialises_like_the_reference():
    import gpb200 as g
    X, ys, _, _ = gpa_problem()
    k = g.SEIso(0.0, 0.0)
    gp = g.GP(X.T, ys["BernLik"], g.MeanZero(), k, g.BernLik(), engine=StubEngine(k))
    assert isinstance(gp, g.GPA) and np.all(gp.v == 0)
    assert gp._eng.calls[-1] == ("factorize", -400.0, 1e-6)           # PDMat(Σ + 1e-6 I), GPA.jl:105
    o = go.update_target(("SEIso", [0.0, 0.0]), X, ys["BernLik"], ("MeanZero",), ("BernLik",), np.zeros(20), init=True)
    assert abs(gp.target - o["target"]) <= 1e-12 * abs(o["target"])
    gp.update_target()
    assert gp._eng.calls[-1] == ("factorize", -20.0, 0.0)             # update_cK!(::GPA), GPA.jl:111-114


@pytest.mark.parametrize("name", LIKS)
def test_gradient_order_matches_the_oracle(name):
    gp, X, y, rng = _stub_gpa(name)
    hyp = gp.get_params()
    assert hyp.size == gp.num_params() == 30 + gp.lik.num_params() + 1 + 3
    hyp = hyp + 0.3 * rng.standard_normal(hyp.size)
    gp.set_params(hyp)
    assert np.allclose(gp.get_params(), hyp, rtol=1e-14, atol=1e-15)      # round trip (lσ is stored as σ, as in the reference)
    gp.update_target_and_dtarget()
    nl = gp.lik.num_params()
    lik = dict(BernLik=("BernLik",), BinLik=("BinLik", 30), ExpLik=("ExpLik",), PoisLik=("PoisLik",),
               GaussLik=("GaussLik", hyp[30] if nl else 0), StuTLik=("StuTLik", 3, hyp[30] if nl else 0))[name]
    spec = gp.kernel.spec()
    o = go.update_dll(spec, X, y, ("MeanConst", hyp[30 + nl]), lik, hyp[:30])
    assert abs(gp.target - o["target"]) <= 1e-12 * abs(o["target"])
    assert np.allclose(gp.dtarget, o["dtarget"], rtol=1e-10, atol=1e-12)


def test_gradient_flags_select_blocks():
    gp, X, y, _ = _stub_gpa("StuTLik")
    gp.update_target_and_dtarget()
    full = gp.dtarget.copy()
    n, nl, nm, nk = 30, 1, 1, 3
    for kw, sl in [(dict(process=False), slice(n, None)), (dict(lik=False), np.r_[0:n, n + nl:n + nl + nm + nk]),
                   (dict(domean=False), np.r_[0:n + nl, n + nl + nm:n + nl + nm + nk]), (dict(kern=False), slice(0, n + nl + nm))]:
        gp.update_target_and_dtarget(**kw)
        assert np.allclose(gp.dtarget, full[sl], rtol=1e-12, atol=1e-14), kw
    gp._eng.calls.clear()
    gp.update_dtarget(process=False, kern=False)
    assert not any(c[0] == "gpa_grad" for c in gp._eng.calls)           # no device gradient needed
    gp.update_target(kern=False)
    assert not any(c[0] == "factorize" for c in gp._eng.calls)          # update_ll!(kern=false) keeps cK
    gp.update_target_and_dtarget(kern=False)
    assert gp._eng.calls[-1] == ("gpa_grad", True, False)
    with pytest.raises(ValueError):
        gp.set_params(np.zeros(3))


def test_set_params_with_flags():
    gp, _, _, _ = _stub_gpa("GaussLik")
    gp.set_params(np.arange(30.0), lik=False, domean=False, kern=False)
    assert np.array_equal(gp.v, np.arange(30.0))
    gp.set_params([0.7, 0.1, 0.2, 0.3], process=False, domean=False)
    assert np.isclose(gp.lik.get_params()[0], 0.7, rtol=1e-15) and gp.kernel.get_params() == [0.1, 0.2, 0.3]


def test_bad_y_is_rejected():
    import gpb200 as g
    X, _, _, _ = gpa_problem()
    k = g.SEIso(0.0, 0.0)
    bad = [(g.BernLik(), np.zeros(20)), (g.BernLik(), np.arange(20)), (g.BinLik(5), np.full(20, 6)), (g.BinLik(5), np.full(20, 1.0)),
           (g.PoisLik(), -np.ones(20, dtype=np.int64)), (g.PoisLik(), np.full(20, 0.5)), (g.ExpLik(), np.zeros(20, dtype=bool)),
           (g.GaussLik(0.0), np.zeros(19))]
    for lik, y in bad:
        with pytest.raises(ValueError):
            g.GPA(X.T, y, g.MeanZero(), k, lik, engine=StubEngine(k))
    with pytest.raises(ValueError):
        g.GPA(X.T, np.zeros(20), g.MeanZero(), k, None, engine=StubEngine(k))


def test_quadrature_predict_obs_matches_the_closed_forms():
    import gpb200 as g
    from gpb200.likelihoods import Likelihood
    rng = np.random.default_rng(4)
    m, s2 = rng.standard_normal(50), rng.random(50) * 2
    for lik in (g.GaussLik(-0.3), g.BernLik()):
        mq, vq = Likelihood.predict_obs(lik, m, s2)                     # the generic 20-node rule on the same likelihood
        mc, vc = lik.predict_obs(m, s2)
        assert np.allclose(mq, mc, rtol=1e-4, atol=1e-4) and np.allclose(vq, vc, rtol=1e-3, atol=1e-4)
    mq, vq = Likelihood.predict_obs(g.GaussLik(-0.3), m, s2)
    assert np.allclose(mq, m, rtol=1e-12) and np.allclose(vq, s2 + math.exp(-0.6), rtol=1e-10)
    for name, lik, tl in [("ExpLik", g.ExpLik(), ("ExpLik",)), ("PoisLik", g.PoisLik(), ("PoisLik",)), ("BinLik", g.BinLik(7), ("BinLik", 7)),
                          ("StuTLik", g.StuTLik(4, 0.2), ("StuTLik", 4, 0.2))]:
        a, b = lik.predict_obs(m, s2), go.predict_obs(tl, m, s2)
        assert np.allclose(a[0], b[0], rtol=1e-13) and np.allclose(a[1], b[1], rtol=1e-12, atol=1e-14), name


def test_host_likelihoods_match_the_oracle():
    import gpb200 as g
    X, ys, liks, rng = gpa_problem(n=40)
    f = rng.standard_normal(40)
    objs = dict(BernLik=g.BernLik(), BinLik=g.BinLik(40), ExpLik=g.ExpLik(), GaussLik=g.GaussLik(-1.0), PoisLik=g.PoisLik(),
                StuTLik=g.StuTLik(3, 0.1))
    for name in LIKS:
        lik, tl, y = objs[name], liks[name], objs[name].check_y(ys[name])
        assert np.allclose(lik.log_dens(f, y), go.log_dens(tl, f, y), rtol=1e-13, atol=1e-14), name
        assert np.allclose(lik.dlog_dens_df(f, y), go.dlog_dens_df(tl, f, y), rtol=1e-13, atol=1e-14), name
        assert np.allclose(lik.dlog_dens_dθ(f, y), go.dlog_dens_dθ(tl, f, y), rtol=1e-13, atol=1e-14), name


def test_host_predictions_match_the_oracle():
    gp, X, y, rng = _stub_gpa("PoisLik")
    gp.set_params(gp.get_params() + 0.2 * rng.standard_normal(gp.num_params()))
    gp.update_target()
    Xs = 2 * np.pi * rng.random((25, 3))
    o = go.update_target(gp.kernel.spec(), X, y, gp.mean.spec(), ("PoisLik",), gp.v)
    mu, s2 = gp.predict_f(Xs.T)
    mo, so = go.predict_f(gp.kernel.spec(), X, gp.mean.spec(), o, Xs)
    assert np.allclose(mu, mo, rtol=1e-9, atol=1e-12) and np.allclose(s2, so, rtol=1e-8, atol=1e-12)
    my, vy = gp.predict_y(Xs.T)
    mo, vo = go.predict_y(gp.kernel.spec(), X, gp.mean.spec(), ("PoisLik",), o, Xs)
    assert np.allclose(my, mo, rtol=1e-8) and np.allclose(vy, vo, rtol=1e-8)


def test_julia_shim_binds_the_gpa_entry_points():
    src = open(os.path.join(ROOT, "gaussianprocesses.jl_b200", "julia", "GPB200.jl")).read()
    assert "ccall((:gpb200_unwhiten, LIB)" in src and "ccall((:gpb200_gpa_grad, LIB)" in src
    assert re.search(r"mutable struct B200GPA\{[^}]*\} <: GPBase", src)
    for fn in ("update_target!", "update_target_and_dtarget!", "get_params", "set_params!", "num_params", "predict_y"):
        assert re.search(r"function (GaussianProcesses\.)?%s\(gp::B200GPA" % re.escape(fn), src), fn
