"""The sparse restatement of the predictive gradients (xgrad_oracle.fitc_predict_f_grad) against central differences of
gp_oracle.fitc_predict's mean and unclamped variance, for FITC, DTC and SoR."""
import numpy as np
import pytest
import scipy.linalg as sl

from conftest import kernel_zoo, make_data
from oracle import gp_oracle as orc
import xgrad_oracle as xo


def _pf(spec, Xu, f, Xs, mspec):
    Kux = orc.cov(spec, Xu, Xs)
    mu = orc.mean_and_grads(mspec, Xs)[0] + Kux.T @ f["alpha_u"]
    q = np.sum(sl.solve_triangular(f["Uuu"], Kux, trans="T", lower=False) ** 2, axis=0)
    s = np.sum(sl.solve_triangular(f["Us"], Kux, trans="T", lower=False) ** 2, axis=0)
    return mu, (s if f["mode"] == "SoR" else np.diag(orc.cov(spec, Xs, Xs)) - q + s)


@pytest.mark.parametrize("mode", ["FITC", "DTC", "SoR"])
@pytest.mark.parametrize("name", ["SEIso", "Mat32Ard", "SE*RQ", "LinIso+Const", "Masked"])
def test_fitc_xgrad_oracle_fd(mode, name):
    spec = dict(kernel_zoo(3))[name].spec()
    X, y, Xs = make_data(80, 3, 9, m=7)
    Xu = X[::8].copy()
    mspec = ("MeanConst", 0.2)
    f = orc.fitc_fit(spec, X, Xu, y, -1.0, mspec, mode=mode)
    mu, var, dmu, dvar = xo.fitc_predict_f_grad(spec, X, Xu, f, Xs, mspec)
    mo, vo = _pf(spec, Xu, f, Xs, mspec)
    np.testing.assert_allclose(mu, mo, rtol=0, atol=1e-12 * np.max(np.abs(mo)))
    np.testing.assert_allclose(var, vo, rtol=0, atol=1e-12 * np.max(np.abs(vo)) + 1e-14)
    h = 1e-5
    for p in range(3):
        E = np.zeros_like(Xs); E[:, p] = h
        (mp, vp), (mm, vm) = _pf(spec, Xu, f, Xs + E, mspec), _pf(spec, Xu, f, Xs - E, mspec)
        assert np.max(np.abs(dmu[:, p] - (mp - mm) / (2 * h))) <= 1e-6 * max(np.max(np.abs(dmu)), 1.0)
        assert np.max(np.abs(dvar[:, p] - (vp - vm) / (2 * h))) <= 1e-6 * max(np.max(np.abs(dvar)), 1e-3)
