"""GPU: GPA (src/GPA.jl) on the device against tests/gpa_oracle.py -- unwhiten, target, the process and kernel gradients for
all six likelihoods and three kernels (single SEIso: the TMA trace kernel; two composites: the kernel-program one), finite
differences of the device target, bitwise reproducibility, predictions, the handle state after gpb200_gpa_grad, error codes
and launch counts.  The GPA nugget is only exp(-40), so the kernels are chosen well conditioned and every bound scales
with the measured cond(K) * eps."""
import ctypes as C
import functools
import json

import numpy as np
import pytest

import gpa_oracle as go

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
LIKS = ["BernLik", "BinLik", "ExpLik", "GaussLik", "PoisLik", "StuTLik"]


def _kernel(name):
    import gpb200 as g
    return dict(SEIso=lambda: g.SEIso(-2.5, 0.0),
                SE_Noise=lambda: g.SEIso(-0.5, 0.1) + g.Noise(-1.0),
                Mat32xRQ_Noise=lambda: g.Mat32Iso(-0.3, 0.1) * g.RQIso(0.2, -0.2, 0.3) + g.Noise(-0.8))[name]()


def _problem(n, seed=1, d=3):
    """test/gpa.jl:8-20"""
    rng = np.random.default_rng(seed)
    X = 2 * np.pi * rng.random((n, d))
    f = np.sin(X).sum(axis=1) / d
    ys = dict(BernLik=rng.random(n) < np.abs(f), BinLik=rng.binomial(n, np.exp(f) / (1 + np.exp(f))).astype(np.int64),
              ExpLik=rng.exponential(f ** 2), GaussLik=f.copy(), PoisLik=rng.poisson(np.exp(f)).astype(np.int64),
              StuTLik=f + rng.standard_t(3, n))
    return X, ys, rng


def _liks(name, n):
    import gpb200 as g
    obj = dict(BernLik=g.BernLik(), BinLik=g.BinLik(n), ExpLik=g.ExpLik(), GaussLik=g.GaussLik(-1.0), PoisLik=g.PoisLik(),
               StuTLik=g.StuTLik(3, 0.1))[name]
    return obj


def _lik_tuple(gp):
    lk = gp.lik
    name = type(lk).__name__
    return dict(BernLik=("BernLik",), BinLik=("BinLik", getattr(lk, "n", 0)), ExpLik=("ExpLik",), PoisLik=("PoisLik",),
                GaussLik=("GaussLik", lk.get_params()[0] if lk.num_params() else 0),
                StuTLik=("StuTLik", getattr(lk, "nu", 0), lk.get_params()[0] if lk.num_params() else 0))[name]


@functools.lru_cache(maxsize=None)
def _cond(kname, n, seed=1):
    from oracle.gp_oracle import cov
    X, _, _ = _problem(n, seed)
    w = np.linalg.eigvalsh(cov(_kernel(kname).spec(), X) + np.exp(-40.0) * np.eye(n))
    return w[-1] / w[0]


def _gpa(lname, kname, n, seed=1):
    import gpb200 as g
    X, ys, rng = _problem(n, seed)
    gp = g.GPA(X.T, ys[lname], g.MeanConst(0.1), _kernel(kname), _liks(lname, n))
    p = gp.get_params()
    p[:n] = 0.5 * rng.standard_normal(n)
    p[n:n + gp.lik.num_params()] += 0.3 * rng.standard_normal(gp.lik.num_params())
    gp.set_params(p)
    return gp, X, ys[lname], rng


def _oracle(gp, X, y, method):
    return go.update_dll(gp.kernel.spec(), X, y, gp.mean.spec(), _lik_tuple(gp), gp.v, method=method)


def test_unwhiten_is_L_times_v():
    import gpb200 as g
    X, _, rng = _problem(700)
    eng = g.Engine(0)
    eng.set_data(X)
    k = _kernel("SE_Noise")
    ops, dims, theta, _ = g.flatten(k, 3)
    eng.set_kernel(ops, dims, theta.size)
    eng.factorize(theta, -20.0)
    v = rng.standard_normal(700)
    L = eng.factor_upper().T
    f = eng.unwhiten(v)
    assert np.max(np.abs(f - L @ v)) <= 1e-13 * np.max(np.abs(L @ v))
    assert np.array_equal(f, eng.unwhiten(v))
    eng.close()


@pytest.mark.parametrize("n", [20, 700, 3000])
@pytest.mark.parametrize("kname", ["SEIso", "SE_Noise", "Mat32xRQ_Noise"])
@pytest.mark.parametrize("lname", LIKS)
def test_target_and_gradients_match_the_oracle(lname, kname, n):
    gp, X, y, _ = _gpa(lname, kname, n)
    gp.update_target_and_dtarget()
    o = _oracle(gp, X, y, "literal" if n <= 700 else "closed")
    bound = 50.0 * _cond(kname, n) * EPS * max(n, 100)
    assert abs(gp.target - o["target"]) <= bound * max(1.0, abs(o["target"])), (gp.target, o["target"])
    nk = gp.kernel.num_params()
    for part, sl in (("process", slice(0, n)), ("kernel", slice(gp.dtarget.size - nk, None)), ("all", slice(None))):
        a, b = gp.dtarget[sl], o["dtarget"][sl]
        err = np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)
        assert err <= bound, (part, err, bound)


@pytest.mark.parametrize("lname", ["BernLik", "StuTLik", "GaussLik"])
def test_directional_finite_differences_of_the_device_target(lname):
    gp, X, y, rng = _gpa(lname, "Mat32xRQ_Noise", 700)
    p0 = gp.get_params()
    gp.update_target_and_dtarget()
    g0 = gp.dtarget.copy()
    for _ in range(2):
        e = rng.standard_normal(p0.size)
        e /= np.linalg.norm(e)
        h = 1e-5
        t = []
        for s in (1, -1):
            gp.set_params(p0 + s * h * e)
            gp.update_target()
            t.append(gp.target)
        gp.set_params(p0)
        fd = (t[0] - t[1]) / (2 * h)
        assert abs(fd - g0 @ e) <= 1e-6 * (np.linalg.norm(g0) + abs(fd)), (fd, g0 @ e)


def test_two_calls_are_bitwise_equal():
    gp, _, _, _ = _gpa("PoisLik", "SEIso", 3000)
    gp.update_target_and_dtarget()
    a, ta = gp.dtarget.copy(), gp.target
    gp.update_target_and_dtarget()
    assert np.array_equal(a, gp.dtarget) and ta == gp.target
    gp2, _, _, _ = _gpa("PoisLik", "Mat32xRQ_Noise", 3000)
    gp2.update_target_and_dtarget()
    b = gp2.dtarget.copy()
    gp2.update_target_and_dtarget()
    assert np.array_equal(b, gp2.dtarget)


@pytest.mark.parametrize("lname", ["BernLik", "PoisLik", "StuTLik"])
def test_predictions_match_the_oracle(lname):
    gp, X, y, rng = _gpa(lname, "SE_Noise", 700)
    gp.update_target()
    Xs = 2 * np.pi * rng.random((300, 3))
    o = go.update_target(gp.kernel.spec(), X, y, gp.mean.spec(), _lik_tuple(gp), gp.v)
    bound = 50.0 * _cond("SE_Noise", 700) * EPS * 700
    mu, s2 = gp.predict_f(Xs.T)
    mo, so = go.predict_f(gp.kernel.spec(), X, gp.mean.spec(), o, Xs)
    assert np.max(np.abs(mu - mo)) <= bound * np.max(np.abs(mo)) and np.max(np.abs(s2 - so)) <= bound * np.max(np.abs(so))
    my, vy = gp.predict_y(Xs.T)
    mo2, vo2 = go.predict_y(gp.kernel.spec(), X, gp.mean.spec(), _lik_tuple(gp), o, Xs)
    assert np.allclose(my, mo2, rtol=1e3 * bound, atol=1e3 * bound) and np.allclose(vy, vo2, rtol=1e3 * bound, atol=1e3 * bound)
    mc, cc = gp.predict_f(Xs[:100].T, full_cov=True)
    moc, coc = go.predict_f(gp.kernel.spec(), X, gp.mean.spec(), o, Xs[:100], full_cov=True)
    assert np.max(np.abs(cc - coc)) <= bound * np.max(np.abs(coc))
    z_rng = np.random.default_rng(9)
    draws = gp.rand(Xs[:100].T, n=4, nugget=1e-6, rng=np.random.default_rng(9))
    z = z_rng.standard_normal((4, 100))
    Lc = np.linalg.cholesky(coc + 1e-6 * np.eye(100))
    ref = (moc[None, :] + z @ Lc.T).T
    assert np.max(np.abs(draws - ref)) <= 1e-6 * np.max(np.abs(ref))
    gp.update_target_and_dtarget()                                   # the factor survives the gradient
    mu2, _ = gp.predict_f(Xs.T)
    assert np.array_equal(mu, mu2)


def _engine(X, kern, capacity=0):
    import gpb200 as g
    eng = g.Engine(0)
    if capacity:
        eng.set_option("capacity", capacity)
    eng.set_data(X)
    ops, dims, theta, _ = g.flatten(kern, X.shape[1])
    eng.set_kernel(ops, dims, theta.size)
    return eng, theta


def test_state_after_gpa_grad_matches_a_fresh_handle():
    import gpb200 as g
    X, ys, rng = _problem(1100)
    Xold, Xnew, r = X[:900], X[900:], rng.standard_normal(1100)
    k = _kernel("SE_Noise")
    a, theta = _engine(Xold, k, capacity=1100)
    b, _ = _engine(Xold, k, capacity=1100)
    for e in (a, b):
        e.factorize(theta, -20.0)
    v, gg = rng.standard_normal(900), rng.standard_normal(900)
    a.gpa_grad(v, gg)
    with pytest.raises(ValueError):                                  # K^-1 and alpha are gone: ESTATE
        a.grad_kernel()
    with pytest.raises(ValueError):
        a.cv_param(0)
    with pytest.raises(ValueError):
        a.predict(X[:5], None)
    assert a.logdet() == b.logdet() and np.array_equal(a.solve(r[:900]), b.solve(r[:900]))
    for e in (a, b):
        e.mll(r[:900]); e.grad_prepare()
    assert np.array_equal(a.grad_kernel()[0], b.grad_kernel()[0])
    za, zb = a.cv_param(0), b.cv_param(0)
    assert np.array_equal(za[0], zb[0]) and np.array_equal(za[1], zb[1])
    a.gpa_grad(v, gg)
    for e in (a, b):
        e.append(Xnew)
    ma, mb = a.mll(r), b.mll(r)
    assert np.array_equal(ma[0], mb[0]) and ma[1] == mb[1]
    a.close(); b.close()


def test_error_codes():
    import gpb200 as g
    from gpb200 import capi
    X, _, rng = _problem(300)
    eng, theta = _engine(X, _kernel("SE_Noise"))
    v, f = rng.standard_normal(300), np.empty(300)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    assert eng._lib.gpb200_unwhiten(eng._h, dp(v), dp(f)) == capi.ESTATE
    assert eng._lib.gpb200_gpa_grad(eng._h, dp(v), dp(v), dp(f), None) == capi.ESTATE
    eng.factorize(theta, -20.0)
    assert eng._lib.gpb200_unwhiten(eng._h, None, dp(f)) == capi.EINVAL
    assert eng._lib.gpb200_gpa_grad(eng._h, dp(v), None, dp(f), None) == capi.EINVAL
    assert eng._lib.gpb200_gpa_grad(eng._h, dp(v), dp(v), None, None) == capi.OK
    eng.close()
    grp = g.LocalGroupEngine(2, rb=1)
    grp.set_data(X)
    ops, dims, th, _ = g.flatten(_kernel("SE_Noise"), 3)
    grp.set_kernel(ops, dims, th.size)
    grp.factorize(th, -20.0)
    lead = grp.lead
    assert lead._lib.gpb200_unwhiten(lead._h, dp(v), dp(f)) == capi.EINVAL
    assert lead._lib.gpb200_gpa_grad(lead._h, dp(v), dp(v), dp(f), None) == capi.EINVAL
    grp.close()


def _device_kernels(fn, tmp_path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "launches.pt.trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as fh:
        events = json.load(fh)["traceEvents"]
    return sum(1 for e in events if e.get("cat") == "kernel" and not e.get("name", "").startswith(("Memcpy", "Memset")))


@pytest.mark.parametrize("kname", ["SEIso", "Mat32xRQ_Noise"])
def test_launch_counts(kname, tmp_path):
    """the counter's growth over unwhiten / gpa_grad equals the kernels torch.profiler records (as test_gpu_launch_count.py)"""
    gp, X, y, rng = _gpa("BernLik", kname, 1500)
    eng = gp._eng
    dl = rng.standard_normal(1500)
    steps = [("unwhiten", lambda: eng.unwhiten(gp.v)), ("gpa_grad", lambda: eng.gpa_grad(gp.v, dl)),
             ("gpa_grad process", lambda: eng.gpa_grad(gp.v, dl, kern=False)), ("step", gp.update_target_and_dtarget)]
    rows = []
    for name, fn in steps:
        c0 = eng.launch_count()
        kernels = _device_kernels(fn, tmp_path)
        rows.append((name, eng.launch_count() - c0, kernels))
    for name, counted, kernels in rows:
        print("launch count GPA %-14s %-18s counted %6d  device %6d" % (kname, name, counted, kernels))
    assert all(c == k for _, c, k in rows), rows


@pytest.mark.slow
def test_full_size_bernoulli():
    """SEIso + Noise, N = 32768, d = 8, Bernoulli: directional finite differences and bitwise reproducibility"""
    import gpb200 as g
    n, d = 32768, 8
    X, ys, rng = _problem(n, seed=5, d=d)
    gp = g.GPA(X.T, ys["BernLik"], g.MeanConst(0.1), g.SEIso(0.5, 0.0) + g.Noise(-1.0), g.BernLik())
    p0 = gp.get_params()
    p0[:n] = 0.5 * rng.standard_normal(n)
    gp.set_params(p0)
    gp.update_target_and_dtarget()
    g0, t0 = gp.dtarget.copy(), gp.target
    gp.update_target_and_dtarget()
    assert np.array_equal(g0, gp.dtarget) and t0 == gp.target
    for part in (slice(0, n), slice(n, None)):                     # latent block, then the hyper-parameters
        e = np.zeros(p0.size)
        e[part] = rng.standard_normal(e[part].size)
        e /= np.linalg.norm(e)
        h = 1e-4
        t = []
        for s in (1, -1):
            gp.set_params(p0 + s * h * e)
            gp.update_target()
            t.append(gp.target)
        fd = (t[0] - t[1]) / (2 * h)
        assert abs(fd - g0 @ e) <= 1e-5 * (np.linalg.norm(g0[part]) + abs(fd)), (fd, g0 @ e)
    gp.set_params(p0)
