"""The numpy restatement of the predictive gradients (xgrad_oracle) against central differences of the dense oracle's
predict_f, for every kernel of the zoo at d = 1 and d = 3, at test points away from and on training inputs."""
import numpy as np
import pytest
import scipy.linalg as sl

from conftest import kernel_zoo, make_data
from oracle import gp_oracle as orc
import xgrad_oracle as xo

ZOO1 = [n for n, _ in kernel_zoo(1)]
ZOO3 = [n for n, _ in kernel_zoo(3)]
# Where a test point meets an input, Mat12 has no derivative and Noise jumps (k(x, x_i) is the noise variance only at x = x_i,
# so differences around x_i see another function than the one evaluated at x_i, which is what Dual inputs differentiate)
_NOT_SMOOTH_ON_POINTS = ("Mat12", "(SE+Mat12)", "LinArd+Noise")


def _spec(name, d):
    return dict(kernel_zoo(d))[name].spec()


def _fd(spec, X, f, Xs, mspec, h=1e-5):
    """central differences of (mu, var): every test point moves at once, each one's prediction depends on it alone"""
    M, d = Xs.shape
    dmu, dvar = np.empty((M, d)), np.empty((M, d))
    for p in range(d):
        E = np.zeros_like(Xs)
        E[:, p] = h
        mp, vp = _pf(spec, X, f, Xs + E, mspec)
        mm, vm = _pf(spec, X, f, Xs - E, mspec)
        dmu[:, p], dvar[:, p] = (mp - mm) / (2 * h), (vp - vm) / (2 * h)
    return dmu, dvar


def _pf(spec, X, f, Xs, mspec):
    mu, _ = orc.predict_f(spec, X, f, Xs, mspec)
    # the unclamped variance (predict_f clamps at 0, which is flat where it acts)
    V = sl.solve_triangular(f["U"], orc.cov(spec, X, Xs), trans="T", lower=False)
    return mu, np.diag(orc.cov(spec, Xs, Xs)) - np.sum(V * V, axis=0)


def _check(name, d, on_points):
    spec = _spec(name, d)
    X, y, Xs = make_data(60, d, 7, m=9)
    Xs = 0.8 * Xs
    if on_points:
        Xs[:4] = X[[3, 11, 20, 41]]
    mspec = ("MeanLin", [0.3 * (p + 1) for p in range(d)])
    f = orc.fit(spec, X, y, -1.0, mspec)
    mu, var, dmu, dvar = xo.predict_f_grad(spec, X, f, Xs, mspec)
    mo, vo = _pf(spec, X, f, Xs, mspec)
    np.testing.assert_allclose(mu, mo, rtol=0, atol=1e-12 * np.max(np.abs(mo)))
    np.testing.assert_allclose(var, vo, rtol=0, atol=1e-12 * np.max(np.abs(vo)) + 1e-14)
    fmu, fvar = _fd(spec, X, f, Xs, mspec)
    assert np.max(np.abs(dmu - fmu)) <= 1e-6 * max(np.max(np.abs(fmu)), 1.0), (dmu, fmu)
    assert np.max(np.abs(dvar - fvar)) <= 1e-6 * max(np.max(np.abs(fvar)), 1e-3), (dvar, fvar)


@pytest.mark.parametrize("name", ZOO3)
def test_xgrad_oracle_fd_d3(name):
    _check(name, 3, False)


@pytest.mark.parametrize("name", ZOO1)
def test_xgrad_oracle_fd_d1(name):
    _check(name, 1, False)


@pytest.mark.parametrize("name", [n for n in ZOO3 if not n.startswith(_NOT_SMOOTH_ON_POINTS)])
def test_xgrad_oracle_fd_on_training_points(name):
    _check(name, 3, True)


@pytest.mark.parametrize("leaf", ["SEIso", "Mat12Iso", "Mat32Iso", "Mat52Iso", "RQIso", "Periodic", "SEArd", "Mat12Ard",
                                  "Mat32Ard", "Mat52Ard", "RQArd"])
def test_r0_rule_stationary(leaf):
    """at r = 0 every stationary leaf gives a finite derivative, 0 (the limit; Mat12's choice), never NaN"""
    ard = leaf.endswith("Ard")
    theta = {"RQIso": [0.1, 0.2, 0.3], "Periodic": [0.1, 0.2, 0.3], "RQArd": [0.1, -0.2, 0.0, 0.3, 0.1]}.get(
        leaf, [0.1, -0.2, 0.0, 0.3] if ard else [0.1, 0.3])
    X = np.array([[0.3, -0.7, 1.1]])
    spec = (leaf, theta) if leaf != "Periodic" else ("Masked", (leaf, theta), [1])
    K, D = xo.cov_dx(spec, X, X)
    assert np.all(np.isfinite(D)) and np.all(D == 0.0)
    # and the one-sided limit agrees for the smooth ones: a tiny offset gives a tiny derivative
    if not leaf.startswith("Mat12"):
        _, Dh = xo.cov_dx(spec, X + 1e-7, X)
        assert np.max(np.abs(Dh)) < 1e-5


def test_r0_rule_linear_and_constant():
    """Lin and Poly keep their ordinary derivative at r = 0; Noise and Const are 0 everywhere"""
    X = np.array([[0.3, -0.7, 1.1]])
    _, D = xo.cov_dx(("LinIso", [0.2]), X, X)
    np.testing.assert_allclose(D[0, 0], X[0] / np.exp(0.4), rtol=1e-15)
    _, D = xo.cov_dx(("Poly", [0.2, -0.3], 2), X, X)
    c, s2 = np.exp(0.2), np.exp(-0.6)
    np.testing.assert_allclose(D[0, 0], s2 * 2 * (c + X[0] @ X[0]) * X[0], rtol=1e-14)
    for leaf in ("Noise", "Const"):
        _, D = xo.cov_dx((leaf, [0.1]), X, np.vstack([X, X + 1.0]))
        assert np.all(D == 0.0)


def test_kdiag_dx_linear():
    """d k(x, x)/dx = 2 x / l^2 for LinIso, the term the dense variance gradient adds"""
    Xs = np.array([[0.5, -1.0], [2.0, 0.25]])
    np.testing.assert_allclose(xo.kdiag_dx(("LinIso", [0.3]), Xs), 2 * Xs / np.exp(0.6), rtol=1e-15)
