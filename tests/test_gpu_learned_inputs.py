"""GPU: training-input gradients (gpb200_grad_inputs; GPE / ElasticGPE / GPA with inputs=True) against the numpy
restatement in inputs_grad_oracle, the specialised SEIso sweep against the generic one, bitwise repeatability, the state
rules and the state the call must leave alone, row-sharded in-process groups against one GPU, optimize(inputs=True), and
(slow) directional differences of the device mll at N = 32768 and 16384.

The file sorts after test_gpu_launch_count*.py on purpose: torch.profiler records no device activity in a session started
about a minute or more after the process's first profiling session (test_gpu_gpa.py's), and this file runs longer than
that (see test_gpu_tile_kernel_contracts.py)."""
import functools

import numpy as np
import pytest

from conftest import kernel_zoo, make_data
from oracle import gp_oracle as orc
import inputs_grad_oracle as ig

pytestmark = pytest.mark.gpu

LOGNOISE = -1.0
EPS = np.finfo(np.float64).eps


def _mean(d):
    import gpb200 as g
    return g.MeanLin([0.3 * (p + 1) for p in range(d)])


def _rel(got, want):
    return np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-300)


def _oracle(spec, X, y, ln, mspec):
    """dmll/dX from a dense fit (the A of oracle.fit, without mll_and_dmll's hyper-parameter gradients)"""
    f = orc.fit(spec, X, y, ln, mspec)
    Kinv = orc._potrs_upper(f["U"], np.eye(X.shape[0]))
    A = np.outer(f["alpha"], f["alpha"]) - Kinv
    return ig.contract(spec, X, A) + f["alpha"][:, None] * ig.mean_dx(mspec, X), f["Ky"]


def _check_parity(got, want, Ky, what):
    """1e-8 of the largest entry, as the other dense gradients; where cond(K) forces more, cond(K) eps (recorded)"""
    err = _rel(got, want)
    if err <= 1e-8:
        return
    cond = np.linalg.cond(Ky)
    print("grad_inputs parity %s: rel err %.3e at cond(K) = %.3e" % (what, err, cond))
    assert err <= cond * EPS, (what, err, cond)


@functools.lru_cache(maxsize=None)
def _gpe(name, N, d=3):
    import gpb200 as g
    kern = dict(kernel_zoo(d))[name]
    X, y, _ = make_data(N, d, 11)
    gp = g.GPE(X.T, y, _mean(d), kern, LOGNOISE)
    return gp, kern.spec(), X, y


def _dx(gp):
    gp.update_dmll(noise=False, domean=False, kern=False, inputs=True)
    return gp.dmll.reshape(gp.nobs, gp.dim)


@pytest.mark.parametrize("N", [700, 3000])
@pytest.mark.parametrize("name", [n for n, _ in kernel_zoo(3)])
def test_zoo_parity(name, N):
    gp, spec, X, y = _gpe(name, N)
    want, Ky = _oracle(spec, X, y, LOGNOISE, _mean(3).spec())
    _check_parity(_dx(gp), want, Ky, (name, N))


@pytest.mark.parametrize("N", [128, 129, 256, 257])
@pytest.mark.parametrize("name", ["SEIso", "SE*RQ"])
def test_tile_boundaries(name, N):
    import gpb200 as g
    kern = dict(kernel_zoo(2))[name]
    X, y, _ = make_data(N, 2, 13)
    gp = g.GPE(X.T, y, _mean(2), kern, LOGNOISE)
    want, Ky = _oracle(kern.spec(), X, y, LOGNOISE, _mean(2).spec())
    _check_parity(_dx(gp), want, Ky, (name, N))


@pytest.mark.parametrize("d", [1, 3, 8])
def test_fast_equals_generic(d):
    """the SEIso specialisation and the kernel-program sweep on the same resident K^-1"""
    import gpb200 as g
    X, y, _ = make_data(2000, d, 14)
    gp = g.GPE(X.T, y, g.MeanZero(), g.SEIso(0.3, 0.2), LOGNOISE)
    e = gp._eng
    e.grad_prepare()
    fast = e.grad_inputs()
    e.set_option("gram_fast", 0)
    generic = e.grad_inputs()
    e.set_option("gram_fast", 1)
    assert _rel(fast, generic) <= 1e-12, _rel(fast, generic)
    assert np.array_equal(fast, e.grad_inputs())


@pytest.mark.parametrize("name", ["SEIso", "MaunaLoa-like"])
def test_repeated_calls_bitwise(name):
    gp, _, _, _ = _gpe(name, 700)
    a = _dx(gp).copy()
    b = gp._eng.grad_inputs()
    c = gp._eng.grad_inputs()
    assert np.array_equal(b, c)
    assert np.array_equal(a, _dx(gp))


def test_state_rules_and_read_only():
    import gpb200 as g
    from gpb200 import capi
    X, y, _ = make_data(500, 3, 15)
    kern = g.SEIso(0.2, 0.1) + g.RQIso(0.3, 0.0, 0.2)
    a = g.GPE(X.T, y, g.MeanZero(), kern, LOGNOISE)
    b = g.GPE(X.T, y, g.MeanZero(), kern, LOGNOISE)
    e, lib = a._eng, a._eng._lib
    pd = capi._as_dp
    out = np.empty((500, 3))
    assert lib.gpb200_grad_inputs(e._h, None, pd(out)) == capi.ESTATE              # grad_prepare first
    e.grad_prepare()
    assert lib.gpb200_grad_inputs(e._h, None, None) == capi.EINVAL                 # null output
    # a caller's alpha is not kept: every later call behaves as on a handle that never saw grad_inputs
    other = np.random.default_rng(1).standard_normal(500)
    g_other = e.grad_inputs(other)
    assert not np.array_equal(g_other, e.grad_inputs())
    b._eng.grad_prepare()
    assert np.array_equal(e.grad_kernel()[0], b._eng.grad_kernel()[0])
    za, zb = e.cv_param(0), b._eng.cv_param(0)
    assert np.array_equal(za[0], zb[0]) and np.array_equal(za[1], zb[1])
    e.grad_inputs()
    Xs = np.random.default_rng(2).standard_normal((40, 3))
    pa, pb = e.predict(Xs), b._eng.predict(Xs)
    assert np.array_equal(pa[0], pb[0]) and np.array_equal(pa[1], pb[1])
    assert np.array_equal(e.solve(y), b._eng.solve(y))
    assert np.array_equal(e.grad_kernel()[0], b._eng.grad_kernel()[0])
    assert e.timings()["grad_inputs"] > 0.0
    # S state (after gpa_grad with the kernel gradient): alpha must be NULL
    v, dl = np.random.default_rng(3).standard_normal((2, 500))
    e.gpa_grad(v, dl)
    assert lib.gpb200_grad_inputs(e._h, pd(other), pd(out)) == capi.EINVAL
    assert lib.gpb200_grad_inputs(e._h, None, pd(out)) == capi.OK
    e.gpa_grad(v, dl, kern=False)                                                  # leaves G alone: still S
    assert lib.gpb200_grad_inputs(e._h, None, pd(out)) == capi.OK
    a.update_mll()                                                                # refactorised: neither K^-1 nor S
    assert lib.gpb200_grad_inputs(e._h, None, pd(out)) == capi.ESTATE


@pytest.mark.parametrize("lik", ["BernLik", "PoisLik"])
def test_gpa_parity(lik):
    import gpb200 as g
    import gpa_oracle as go
    rng = np.random.default_rng(16)
    N, d = 300, 3
    X = 2 * np.pi * rng.random((N, d))
    y = (rng.random(N) < 0.5) if lik == "BernLik" else rng.poisson(1.0, N)
    kern = g.SEIso(-0.5, 0.1) + g.Noise(-1.0)
    gp = g.GP(X.T, y, g.MeanLin([0.2, -0.1, 0.3]), kern, getattr(g, lik)())
    v = 0.5 * rng.standard_normal(N)
    gp.set_params(np.concatenate([v, gp.get_params()[N:]]))
    gp.update_target_and_dtarget(inputs=True)
    got = gp.dtarget[-N * d:].reshape(N, d)
    want = ig.dtarget_dx(kern.spec(), X, y, gp.mean.spec(), go_lik(lik), v)
    assert _rel(got, want) <= 1e-8, _rel(got, want)
    # the other entries are those of the call without inputs
    d_all = gp.dtarget.copy()
    gp.update_target_and_dtarget()
    assert np.array_equal(gp.dtarget, d_all[:gp.dtarget.size])


def go_lik(name):
    return {"BernLik": ("BernLik",), "PoisLik": ("PoisLik",)}[name]


def test_elastic_after_append_equals_fresh():
    import gpb200 as g
    X, y, _ = make_data(900, 2, 17)
    kern = g.Mat32Iso(0.3, 0.1)
    el = g.ElasticGPE(X[:600].T, y[:600], _mean(2), kern, LOGNOISE, capacity=1000)
    el.append(X[600:].T, y[600:])
    fresh = g.GPE(X.T, y, _mean(2), kern, LOGNOISE)
    assert _rel(_dx(el), _dx(fresh)) <= 1e-9
    # move the inputs in place (N, d and the capacity unchanged): equal to a fresh model at the moved inputs
    p = el.get_params(inputs=True)
    p[-X.size:] += 0.01 * np.random.default_rng(18).standard_normal(X.size)
    el.set_params(p, inputs=True)
    el.update_target(kern=False, noise=False)
    moved = g.GPE(el.x, y, _mean(2), kern, LOGNOISE)
    assert abs(el.mll - moved.mll) <= 1e-9 * abs(moved.mll)
    assert _rel(_dx(el), _dx(moved)) <= 1e-9


def test_optimize_inputs():
    import gpb200 as g
    rng = np.random.default_rng(19)
    N = 40
    Xt = np.linspace(-3, 3, N)[None, :]
    y = np.sin(2 * Xt[0])
    gp = g.GPE(Xt + 0.15 * rng.standard_normal(Xt.shape), y, g.MeanZero(), g.SEIso(-0.5, 0.0), -2.0)
    gp.update_target_and_dtarget(noise=False, domean=False, kern=False, inputs=True)
    mll0, g0 = gp.mll, np.linalg.norm(gp.dtarget)
    gp.optimize(noise=False, domean=False, kern=False, inputs=True, maxiter=30)
    gp.update_target_and_dtarget(noise=False, domean=False, kern=False, inputs=True)
    print("optimize(inputs=True): mll %.6f -> %.6f, |grad| %.3e -> %.3e" % (mll0, gp.mll, g0, np.linalg.norm(gp.dtarget)))
    assert gp.mll > mll0 and np.linalg.norm(gp.dtarget) < g0


@pytest.mark.parametrize("rb", [1, 2, 4])
@pytest.mark.parametrize("R", [2, 3, 4, 8])
def test_sharded_group_equals_single(R, rb):
    import gpb200 as g
    X, y, _ = make_data(4100, 3, 20)
    for kern in (g.SEIso(0.2, 0.1), g.SEIso(0.2, 0.1) * g.RQIso(0.4, 0.0, 0.1)):
        single = g.GPE(X.T, y, _mean(3), kern, LOGNOISE)
        grp = g.LocalGroupEngine(R, rb=rb)
        try:
            gs = g.GPE(X.T, y, _mean(3), kern, LOGNOISE, engine=grp)
            assert all(e.storage_info()["sharded"] for e in grp.engines)
            a, b = _dx(single), _dx(gs).copy()
            assert _rel(b, a) <= 1e-12, (R, rb, _rel(b, a))
            assert np.array_equal(b, grp.grad_inputs() + gs.alpha[:, None] * gs.mean.grad_x(gs._xpm))
            assert np.array_equal(grp.grad_inputs(), grp.grad_inputs())
            if R == 4 and rb == 2:                    # moving the inputs on a group: nothing reallocated, same as one GPU
                p = gs.get_params(inputs=True)
                p[-X.size:] += 0.01
                gs.set_params(p, inputs=True)
                single.set_params(p, inputs=True)
                gs.update_target(kern=False, noise=False)
                single.update_target(kern=False, noise=False)
                assert abs(gs.mll - single.mll) <= 1e-10 * abs(single.mll)
                assert _rel(_dx(gs), _dx(single)) <= 1e-12
        finally:
            grp.close()


def _directional(gp, D, h):
    """sixth-order central difference of the device mll along D (an (N, d) step of the inputs)"""
    p = gp.get_params(inputs=True)
    f = []
    for s in (-3, -2, -1, 1, 2, 3):
        q = p.copy()
        q[p.size - D.size:] += s * h * D.ravel()
        gp.set_params(q, inputs=True)
        gp.update_mll()
        f.append(gp.mll)
    gp.set_params(p, inputs=True)
    gp.update_mll()
    return (-f[0] + 9.0 * f[1] - 45.0 * f[2] + 45.0 * f[3] - 9.0 * f[4] + f[5]) / (60.0 * h)


@pytest.mark.slow
@pytest.mark.parametrize("N,d,which", [(32768, 8, "SEIso"), (16384, 3, "Mat32Iso+RQIso")])
def test_directional_derivative_at_scale(N, d, which):
    import gpb200 as g
    X, y, _ = make_data(N, d, 21)
    X *= 2.0
    kern = g.SEIso(0.5, 0.0) if which == "SEIso" else g.Mat32Iso(0.3, 0.0) + g.RQIso(0.2, -0.5, 0.0)
    gp = g.GPE(X.T, y, g.MeanZero(), kern, -1.0)
    gx = _dx(gp)
    D = np.random.default_rng(22).standard_normal(X.shape)
    dd = float(np.sum(gx * D))
    fds = [_directional(gp, D, h) for h in (1e-3, 3e-4)]
    fd = min(fds, key=lambda v: abs(v - dd))
    rel = abs(dd - fd) / np.linalg.norm(gx)
    print("directional dmll/dX %s N=%d: <g, D> = %.9e, fd = %.9e (%s), rel to |g| %.3e" % (which, N, dd, fd, fds, rel))
    assert rel <= 1e-6
