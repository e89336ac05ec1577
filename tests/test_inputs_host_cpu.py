"""CPU: the host side of the training-input parameters (gpb200/gpe.py, gpb200/gpa.py) over a stand-in engine backed by the CPU
oracles: the [noise; mean; kernel; vec(X)] and [v; lik; mean; kernel; vec(X)] orders and layouts, inputs=False identical to
the protocol without it, set_params(inputs=True) moving X on the engine and forcing a refactorisation, and
optimize(inputs=True) rolling back a rejected (PosDefException) step."""
import numpy as np
import pytest

import gpb200
from gpb200 import capi
from oracle import gp_oracle as orc
import gpa_oracle as go
import inputs_grad_oracle as ig


class StubEngine:
    """the Engine calls GPE / GPA make, computed densely by the oracles -- TEST ONLY"""

    def __init__(self, kernel):
        self.kernel, self.calls, self.reject = kernel, [], None

    def set_data(self, x_pm):
        self.calls.append("set_data")
        self.X = np.array(x_pm, dtype=np.float64)
        self.N, self.d = self.X.shape
        self.factored = False

    def set_kernel(self, ops, dims, n_theta):
        self.n_theta = int(n_theta)

    def set_option(self, key, value):
        pass

    def factorize(self, theta, log_noise, extra_nugget=0.0):
        self.calls.append("factorize")
        if self.reject is not None and self.reject(self.X):
            self.factored = False
            raise capi.PosDefException(1)
        self.spec, self.ln, self.nug = self.kernel.spec(), log_noise, extra_nugget
        K = orc.gram(self.spec, self.X, log_noise, extra_nugget)
        self.L = np.linalg.cholesky(K)
        self.Kinv = np.linalg.inv(K)
        self.factored = True

    def mll(self, r):
        assert self.factored, "mll on a stale factor"
        self.alpha = self.Kinv @ r
        sign, logdet = np.linalg.slogdet(self.L @ self.L.T)
        return self.alpha.copy(), float(-(r @ self.alpha + logdet + orc.LOG2PI * self.N) / 2)

    def grad_prepare(self):
        self.calls.append("grad_prepare")
        self.A = np.outer(self.alpha, self.alpha) - self.Kinv

    def grad_kernel(self, alpha=None):
        _, grads = orc.cov_and_grads(self.spec, self.X, None, True)
        return np.array([0.5 * np.sum(self.A * G) for G in grads]), float(np.trace(self.A))

    def grad_inputs(self, alpha=None):
        self.calls.append("grad_inputs")
        return ig.contract(self.spec, self.X, self.A)

    def unwhiten(self, v):
        return self.L @ v

    def gpa_grad(self, v, dl_df, process=True, kern=True):
        self.calls.append("gpa_grad")
        self.A = go.S_closed(self.L, dl_df, v)
        _, grads = orc.cov_and_grads(self.spec, self.X, None, True)
        return (self.L.T @ dl_df if process else None), (np.array([0.5 * np.sum(self.A * G) for G in grads]) if kern else None)


def _gpe(n=14, d=2, seed=0, mean=None, kernel=None):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((d, n))
    y = np.sin(X.sum(axis=0)) + 0.1 * rng.standard_normal(n)
    kernel = kernel or gpb200.SEIso(0.2, 0.1)
    eng = StubEngine(kernel)
    gp = gpb200.GPE(X, y, mean or gpb200.MeanLin([0.3, -0.4]), kernel, -1.0, engine=eng)
    return gp, eng


def test_gpe_order_and_layout():
    gp, eng = _gpe()
    base = gp.get_params()
    p = gp.get_params(inputs=True)
    assert p.size == base.size + gp.dim * gp.nobs == gp.num_params(inputs=True)
    assert np.array_equal(p[:base.size], base)
    assert np.array_equal(p[base.size:].reshape(gp.nobs, gp.dim), gp.x.T)        # vec of the dim x nobs matrix
    gp.update_target_and_dtarget()
    d0 = gp.dtarget.copy()
    gp.update_target_and_dtarget(inputs=True)
    assert np.array_equal(gp.dtarget[:d0.size], d0)
    spec, mspec = gp.kernel.spec(), gp.mean.spec()
    want = ig.dmll_dx(spec, gp.x.T, gp.y, gp.logNoise, mspec)
    assert np.allclose(gp.dtarget[d0.size:].reshape(gp.nobs, gp.dim), want, rtol=1e-9, atol=1e-12)


def test_gpe_inputs_false_unchanged():
    gp, eng = _gpe()
    gp.update_target_and_dtarget()
    assert "grad_inputs" not in eng.calls
    assert gp.dtarget.size == gp.num_params()


def test_gpe_only_inputs():
    gp, eng = _gpe()
    gp.update_target_and_dtarget(noise=False, domean=False, kern=False, inputs=True)
    assert gp.dtarget.size == gp.dim * gp.nobs
    want = ig.dmll_dx(gp.kernel.spec(), gp.x.T, gp.y, gp.logNoise, gp.mean.spec())
    assert np.allclose(gp.dtarget.reshape(gp.nobs, gp.dim), want, rtol=1e-9, atol=1e-12)


def test_gpe_set_params_round_trip_and_refactorises():
    gp, eng = _gpe()
    p = gp.get_params(inputs=True)
    q = p.copy()
    q[-gp.dim * gp.nobs:] += 0.01 * np.arange(gp.dim * gp.nobs)
    gp.set_params(q, inputs=True)
    assert np.array_equal(gp.get_params(inputs=True), q)
    assert np.array_equal(eng.X, gp.x.T) and eng.calls[-1] == "set_data"
    n_fact = eng.calls.count("factorize")
    gp.update_target(kern=False, noise=False)               # the factor belongs to the old inputs: refactorised anyway
    assert eng.calls.count("factorize") == n_fact + 1
    assert abs(gp.mll - orc.fit(gp.kernel.spec(), gp.x.T, gp.y, -1.0, gp.mean.spec())["mll"]) < 1e-10
    gp.update_target(kern=False, noise=False)               # and only once
    assert eng.calls.count("factorize") == n_fact + 1
    with pytest.raises(ValueError):
        gp.set_params(q[:-1], inputs=True)


def test_gpe_optimize_rolls_back_rejected_inputs():
    gp, eng = _gpe(n=10)
    x0 = gp.x.copy()
    # a step that moves point 0 far from where it starts is "singular"
    eng.reject = lambda X: np.linalg.norm(X[0] - x0[:, 0]) > 0.05
    before = gp.mll
    res = gp.optimize(inputs=True, maxiter=5)
    assert np.linalg.norm(gp.x[:, 0] - x0[:, 0]) <= 0.05
    assert gp.mll >= before - 1e-12 and np.isfinite(res.fun)


def test_gpa_order_and_value():
    rng = np.random.default_rng(2)
    n, d = 12, 2
    X = 2 * np.pi * rng.random((d, n))
    y = rng.random(n) < 0.5
    kernel = gpb200.SEIso(0.2, 0.1)
    eng = StubEngine(kernel)
    gp = gpb200.GP(X, y, gpb200.MeanLin([0.3, -0.2]), kernel, gpb200.BernLik(), engine=eng)
    v = 0.5 * rng.standard_normal(n)
    gp.set_params(np.concatenate([v, gp.get_params()[n:]]))
    base = gp.get_params()
    p = gp.get_params(inputs=True)
    assert p.size == gp.num_params(inputs=True) == base.size + n * d
    assert np.array_equal(p[base.size:].reshape(n, d), gp.x.T)
    gp.update_target_and_dtarget()
    d0 = gp.dtarget.copy()
    gp.update_target_and_dtarget(inputs=True)
    assert np.array_equal(gp.dtarget[:d0.size], d0)
    want = ig.dtarget_dx(kernel.spec(), gp.x.T, y, gp.mean.spec(), ("BernLik",), v)
    assert np.allclose(gp.dtarget[d0.size:].reshape(n, d), want, rtol=1e-8, atol=1e-11)
    # set_params(inputs=True): moved on the engine, refactorised by update_ll even with kern=False
    q = p.copy()
    q[-n * d:] += 0.02
    gp.set_params(q, inputs=True)
    assert np.array_equal(eng.X, gp.x.T)
    nf = eng.calls.count("factorize")
    gp.update_target(kern=False)
    assert eng.calls.count("factorize") == nf + 1
