"""CPU: the dense restatement of the training-input gradients (inputs_grad_oracle) against fourth-order central differences
of the oracle mll (gp_oracle.fit) and GPA target (gpa_oracle.update_target at fixed v) in every coordinate of X: the kernel
zoo at d = 1 and d = 3, an x-dependent mean, per-point noise, all six GPA likelihoods, and duplicated training inputs."""
import numpy as np
import pytest

from conftest import kernel_zoo, make_data
import inputs_grad_oracle as ig
from test_gpa_cpu import LIKS, gpa_problem

ZOO1 = [n for n, _ in kernel_zoo(1)]
ZOO3 = [n for n, _ in kernel_zoo(3)]
# smooth where two inputs coincide: no Mat12 kink at r = 0, no Noise jump
SMOOTH = ["SEIso", "SEArd", "Mat52Iso", "RQIso", "SE*RQ", "Poly", "LinIso+Const", "Periodic(1d)"]


def _spec(name, d):
    return dict(kernel_zoo(d))[name].spec()


def _check(g, fd_of_h):
    """the closest of three steps: rounding of the mll grows with cond(K), truncation with the kernel's curvature"""
    scale = max(np.max(np.abs(g)), 1e-3)
    err = np.inf
    for h in (1e-3, 3e-4, 1e-4):
        err = min(err, np.max(np.abs(g - fd_of_h(h))))
        if err <= 1e-6 * scale:
            break
    assert err <= 1e-6 * scale, (err, scale)


@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("name", ZOO3)
def test_dmll_dx_fd_zoo(name, d):
    if name not in ZOO1 and d == 1:
        pytest.skip("not in the d = 1 zoo")
    X, y, _ = make_data(24, d, 21 + d)
    spec = _spec(name, d)
    g = ig.dmll_dx(spec, X, y, -1.0)
    assert g.shape == X.shape and np.all(np.isfinite(g))
    _check(g, lambda h: ig.fd_dmll_dx(spec, X, y, -1.0, h=h))


@pytest.mark.parametrize("name", ["SEIso", "Poly", "Masked"])
def test_dmll_dx_fd_linear_mean(name):
    d = 3
    X, y, _ = make_data(20, d, 31)
    spec, mspec = _spec(name, d), ("MeanLin", [0.4, -0.7, 0.2])
    g = ig.dmll_dx(spec, X, y, -1.0, mspec)
    _check(g, lambda h: ig.fd_dmll_dx(spec, X, y, -1.0, mspec, h=h))
    assert np.max(np.abs(g - ig.dmll_dx(spec, X, y, -1.0))) > 1e-3       # the mean's part is not empty


@pytest.mark.parametrize("name", ["SEIso", "LinArd+Noise", "SE*RQ"])
def test_dmll_dx_fd_per_point_noise(name):
    d = 2
    X, y, _ = make_data(20, d, 32)
    ln = np.random.default_rng(4).uniform(-1.5, -0.5, X.shape[0])
    spec = _spec(name, d)
    _check(ig.dmll_dx(spec, X, y, ln), lambda h: ig.fd_dmll_dx(spec, X, y, ln, h=h))


@pytest.mark.parametrize("name", SMOOTH)
def test_dmll_dx_duplicated_inputs(name):
    """two copies of a training input: the stationary leaves give the limit of d1k at r = 0 (0), the gradient stays finite
    and, for kernels differentiable there, matches the finite differences"""
    d = 2
    X, y, _ = make_data(20, d, 33)
    X[7] = X[3]
    spec = _spec(name, d)
    g = ig.dmll_dx(spec, X, y, -1.0)
    assert np.all(np.isfinite(g))
    _check(g, lambda h: ig.fd_dmll_dx(spec, X, y, -1.0, h=h))


def test_dmll_dx_duplicated_inputs_kinked_kernels_finite():
    """Mat12 (kink at r = 0) and the Noise leaf (jump): no derivative exists at a duplicate, the documented convention
    (limit 0 / no contribution) gives finite values"""
    d = 2
    X, y, _ = make_data(20, d, 34)
    X[5] = X[2]
    for name in ("Mat12Iso", "Mat12Ard", "LinArd+Noise", "(SE+Mat12)*RQ"):
        assert np.all(np.isfinite(ig.dmll_dx(_spec(name, d), X, y, -1.0))), name


def test_diagonal_term_is_one_sided():
    """a single point under LinIso: dmll/dx = A_11 d1k(x, x) with d1k = x / l^2, half of d/dx k(x, x)"""
    X, y = np.array([[0.7, -0.2]]), np.array([0.3])
    spec = ("LinIso", [0.1])
    g = ig.dmll_dx(spec, X, y, -1.0)
    _check(g, lambda h: ig.fd_dmll_dx(spec, X, y, -1.0, h=h))
    assert np.max(np.abs(g)) > 1e-3


@pytest.mark.parametrize("name", LIKS)
def test_dtarget_dx_fd_gpa(name):
    X, ys, liks, rng = gpa_problem(n=16, d=2, seed=3)
    y, lik = ys[name], liks[name]
    v = 0.5 * rng.standard_normal(X.shape[0])
    spec, mspec = ("SEIso", [0.2, 0.1]), ("MeanLin", [0.3, -0.2])
    g = ig.dtarget_dx(spec, X, y, mspec, lik, v)
    _check(g, lambda h: ig.fd_dtarget_dx(spec, X, y, mspec, lik, v, h=h))
