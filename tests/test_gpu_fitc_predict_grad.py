"""GPU: predictive gradients of the sparse strategies (gpb200_fitc_predict_grad, FITC / DTC / SoR.predict_f_grad) against
xgrad_oracle.fitc_predict_f_grad at the cond(K_uu) eps bounds of test_gpu_fitc.py, one N above a staging chunk, bitwise
agreement with predict_f, unchanged gradient / CV state, and the error codes (FSA, before mll)."""
import numpy as np
import pytest

from oracle import gp_oracle as orc
import xgrad_oracle as xo

pytestmark = pytest.mark.gpu
EPS = np.finfo(float).eps
MODES = ["FITC", "DTC", "SoR"]


def _kernel(name):
    import gpb200 as g
    return dict(SEIso=lambda: g.SEIso(-0.2, 0.1), SExRQ=lambda: g.SEIso(0.2, 0.1) * g.RQIso(0.3, -0.2, 0.1),
                Mat32=lambda: g.Mat32Ard([0.1, -0.1], 0.0))[name]()


def _problem(mode, kname, N, seed=0):
    import gpb200 as g
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, 2)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-2.5, 2.5, 7)
    Xu = np.array([[a, b] for a in grid for b in grid])
    gp = getattr(g, mode)(X.T, Xu.T, y, g.MeanLin([0.2, -0.1]), _kernel(kname), -1.0)
    return gp, X, Xu, y


def _rel(got, want):
    return np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-300)


@pytest.mark.parametrize("N", [3000, 40000])
@pytest.mark.parametrize("kname", ["SEIso", "SExRQ", "Mat32"])
@pytest.mark.parametrize("mode", MODES)
def test_sparse_parity(mode, kname, N):
    gp, X, Xu, y = _problem(mode, kname, N)
    spec, mspec = gp.kernel.spec(), gp.mean.spec()
    f = orc.fitc_fit(spec, X, Xu, y, -1.0, mspec, mode=mode)
    Kuu = orc.cov(spec, Xu) + 1e-10 * np.eye(Xu.shape[0])
    w = np.linalg.eigvalsh(Kuu)
    tol = max(1e-8, 64.0 * (w[-1] / w[0]) * EPS)
    Xs = np.random.default_rng(5).uniform(-2.8, 2.8, (130, 2))
    mu, s2, dmu, ds2 = gp.predict_f_grad(Xs.T)
    wmu, wvar, wdmu, wdvar = xo.fitc_predict_f_grad(spec, X, Xu, f, Xs, mspec)
    assert dmu.shape == (2, 130) and ds2.shape == (2, 130)
    pm, ps2 = gp.predict_f(Xs.T)
    assert np.array_equal(mu, pm) and np.array_equal(s2, ps2)
    e_mu, e_dmu = _rel(dmu.T, wdmu), _rel(ds2.T[wvar > 0], wdvar[wvar > 0])
    print("%s %s N=%d: dmu %.2e dvar %.2e (bound %.1e)" % (mode, kname, N, e_mu, e_dmu, tol))
    assert e_mu <= tol and e_dmu <= tol


@pytest.mark.parametrize("mode", MODES)
def test_sparse_repeated_and_dmu_only(mode):
    gp, _, _, _ = _problem(mode, "SExRQ", 2000)
    Xs = np.random.default_rng(6).uniform(-2.8, 2.8, (300, 2))
    a, b = gp._eng.predict_grad(Xs), gp._eng.predict_grad(Xs)
    c = gp._eng.predict_grad(Xs, want_var=False)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[2], c[2]) and c[1] is None and c[3] is None


def test_sparse_state_unchanged():
    """kernel gradient, noise gradient and cv_param of the sparse engine are bitwise the same with and without an
    intervening predict_grad (which fills the sub-engines' F upper tiles with L')"""
    Xs = np.random.default_rng(7).uniform(-2.8, 2.8, (100, 2))
    out = []
    for pg in (True, False):
        gp, _, _, _ = _problem("FITC", "SExRQ", 2000)
        e, r = [], []
        if pg:
            gp._eng.predict_grad(Xs)
        r.append(gp._eng.grad_kernel())
        if pg:
            gp._eng.predict_grad(Xs)
        r.append(gp._eng.grad_noise())
        r.extend(gp._eng.cv_param(0))
        if pg:
            gp._eng.predict_grad(Xs)
        r.extend(gp._eng.cv_param(1))
        r.append(gp._eng.predict(Xs)[1])
        out.append(r)
    for u, v in zip(*out):
        assert np.array_equal(np.asarray(u), np.asarray(v))


def test_sparse_errors():
    import gpb200 as g
    from gpb200 import capi
    gp, X, Xu, y = _problem("FITC", "SEIso", 500)
    e = gp._eng
    xs = np.zeros((4, 2))
    with pytest.raises(ValueError, match="single GPU|var and dvar"):
        e._check(e._lib.gpb200_fitc_predict_grad(e._h, 4, capi._as_dp(xs), 2, capi._as_dp(np.empty(4)), capi._as_dp(np.empty(4)),
                                                 capi._as_dp(np.empty((4, 2))), None), "fitc_predict_grad")
    assert e._lib.gpb200_fitc_predict_grad(None, 4, capi._as_dp(xs), 2, None, None, None, None) == capi.EINVAL
    assert e._lib.gpb200_fitc_predict_grad(e._h, 0, capi._as_dp(xs), 2, capi._as_dp(np.empty(4)), None,
                                           capi._as_dp(np.empty((4, 2))), None) == capi.EINVAL
    fresh = capi.FitcEngine(0)
    assert fresh._lib.gpb200_fitc_predict_grad(fresh._h, 4, capi._as_dp(xs), 2, capi._as_dp(np.empty(4)), None,
                                               capi._as_dp(np.empty((4, 2))), None) == capi.ESTATE
    fresh.close()
    order = np.argsort(X[:, 0])
    fsa = g.FSA(X.T, Xu.T, [np.sort(order[i:i + 100]) for i in range(0, 500, 100)], y, g.MeanZero(), _kernel("SEIso"), -1.0)
    with pytest.raises(ValueError, match="FSA"):
        fsa.predict_f_grad(xs.T)
    fe = fsa._eng
    assert fe._lib.gpb200_fitc_predict_grad(fe._h, 4, capi._as_dp(xs), 2, capi._as_dp(np.empty(4)), None,
                                            capi._as_dp(np.empty((4, 2))), None) == capi.EINVAL
