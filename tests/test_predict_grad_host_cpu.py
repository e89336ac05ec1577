"""CPU: the host side of predict_f_grad with a stub engine -- the mean's gradient, GP.jl:75's clamp and the (dim, M) layout."""
import numpy as np
import pytest

import gpb200 as g
from gpb200.gpe import _predict_f_grad


class _StubEngine:
    def __init__(self, var):
        self.var = np.asarray(var, dtype=np.float64)

    def predict_grad(self, xs, alpha=None, want_var=True):
        M, d = xs.shape
        dmu = np.arange(M * d, dtype=np.float64).reshape(M, d)
        return np.ones(M), self.var.copy(), dmu, -dmu - 1.0


def test_mean_gradients():
    X = np.random.default_rng(1).standard_normal((5, 3))
    assert np.array_equal(g.MeanZero().grad_x(X), np.zeros((5, 3)))
    assert np.array_equal(g.MeanConst(0.4).grad_x(X), np.zeros((5, 3)))
    assert np.array_equal(g.MeanLin([1.0, 2.0, 3.0]).grad_x(X), np.tile([1.0, 2.0, 3.0], (5, 1)))

    class _NewMean(g.Mean):                       # a mean without its own grad_x must not pass for a constant one
        def mean(self, X):
            return X[:, 0] ** 2
    with pytest.raises(NotImplementedError):
        _NewMean().grad_x(X)


def test_clamp_layout_and_mean():
    """where the variance is clamped at 0 its gradient is 0 (ForwardDiff's max(., 0.0)); outputs are (dim, M)"""
    xs = np.array([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]])
    mean = g.MeanLin([0.5, -2.0])
    mu, s2, dmu, ds2 = _predict_f_grad(_StubEngine([0.3, -1e-12, 0.0]), xs, None, mean)
    np.testing.assert_array_equal(mu, 1.0 + xs @ np.array([0.5, -2.0]))
    np.testing.assert_array_equal(s2, [0.3, 0.0, 0.0])
    assert dmu.shape == (2, 3) and ds2.shape == (2, 3)
    np.testing.assert_array_equal(dmu, (np.arange(6.0).reshape(3, 2) + [0.5, -2.0]).T)
    np.testing.assert_array_equal(ds2, [[-1.0, 0.0, -5.0], [-2.0, 0.0, -6.0]])
