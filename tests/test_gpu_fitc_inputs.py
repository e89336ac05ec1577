"""GPU: dmll/dX of FITC, DTC, SoR and FSA (gpb200_fitc_grad_kernel_inputs) against the dense oracle
(sparse_inputs_grad_oracle.dmll_dx) over the kernel zoo, at M below, at and above one 128-tile, at the staging and FSA tile
edges; the invariants of the joint call and of gpb200_fitc_set_inputs; the error codes; directional derivatives at scale
against central differences of the device mll; and optimize(inputs=True, inducing=True) end to end."""
import ctypes as C

import numpy as np
import pytest

from conftest import kernel_zoo
import inducing_grad_oracle as ig
import sparse_inputs_grad_oracle as sg

pytestmark = pytest.mark.gpu
MODES = ("FITC", "DTC", "SoR", "FSA")
# the linear-feature kernels have rank d + 1 (LinIso + Const) and 10 (degree-2 Poly at d = 3): more inducing points leave
# K_uu singular up to its nugget; Periodic(1d) sees one coordinate only
M_OF = {"LinIso+Const": 3, "Poly": 6, "Periodic(1d)": 4}


def _blocks(N, seed, sizes=(1, 127, 128, 129, 300, 64)):
    """a partition of 0..N-1 into blocks of the given sizes in turn: every padding case of the layout"""
    perm = np.random.default_rng(seed).permutation(N)
    out, i, k = [], 0, 0
    while i < N:
        out.append(np.sort(perm[i:i + sizes[k % len(sizes)]]))
        i += sizes[k % len(sizes)]
        k += 1
    return out


def _model(mode, kernel, X, Xu, y, blocks=None, ln=-1.0, mean=None):
    import gpb200 as g
    mean = g.MeanConst(0.1) if mean is None else mean
    if mode == "FSA":
        return g.FSA(X.T, Xu.T, blocks, y, mean, kernel, ln)
    return getattr(g, mode)(X.T, Xu.T, y, mean, kernel, ln)


def _data(N, d, seed, L=4.0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-L, L, (N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    return X, y


def _compare(gp, X, Xu, y, mode, blocks, tag):
    spec = gp.kernel.spec()
    gp.update_dmll(inputs=True, noise=False, domean=False, kern=False)
    gx = gp.dmll.reshape(X.shape)
    go = sg.dmll_dx(spec, X, Xu, y, gp.logNoise, mode, blocks, mspec=gp.mean.spec())
    _, c_s = ig.conditioning(spec, X, Xu, gp.logNoise, mode, blocks)
    err = np.max(np.abs(gx - go))
    scale = np.max(np.abs(go))
    print("%-44s cond(S_QR) %.2e  max|err| %.3e  max|g| %.3e  rel %.2e" % (tag, c_s, err, scale, err / scale))
    # the bounds of the inducing-point gradient: the same adjoints, whose error follows cond(Sigma_QR)
    assert err <= 1e-6 * scale + 1e-7, tag
    assert err <= max(1e-7, 1e-12 * c_s) * scale, tag


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", [n for n, _ in kernel_zoo(3)])
def test_zoo_parity(mode, name):
    d, N = 3, 700
    X, y = _data(N, d, 1)
    Xu = np.random.default_rng(2).uniform(-3.6, 3.6, (M_OF.get(name, 50), d))
    blocks = _blocks(N, 3) if mode == "FSA" else None
    gp = _model(mode, dict(kernel_zoo(d))[name], X, Xu, y, blocks)
    _compare(gp, X, Xu, y, mode, blocks, "%s %s N=%d M=%d" % (mode, name, N, Xu.shape[0]))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("N", [700, 3000])
@pytest.mark.parametrize("M", [50, 128, 300])
@pytest.mark.parametrize("case", ["SEIso, MeanLin", "Mat32Ard", "SE*RQ, Xu in x"])
def test_sizes_parity(mode, N, M, case):
    import gpb200 as g
    d = 3
    X, y = _data(N, d, N + M, L=7.0)
    name = case.split(",")[0]
    rng = np.random.default_rng(M)
    Xu = X[rng.permutation(N)[:M]].copy() if "Xu in x" in case else rng.uniform(-6.3, 6.3, (M, d))
    blocks = _blocks(N, 4) if mode == "FSA" else None
    mean = g.MeanLin([0.3, -0.2, 0.1]) if "MeanLin" in case else None
    gp = _model(mode, dict(kernel_zoo(d))[name], X, Xu, y, blocks, mean=mean)
    _compare(gp, X, Xu, y, mode, blocks, "%s %s N=%d M=%d" % (mode, case, N, M))


@pytest.mark.parametrize("mode", ("FITC", "DTC", "SoR"))
@pytest.mark.parametrize("N", [127, 128, 129, 257])
def test_row_tile_edges(mode, N):
    import gpb200 as g
    X, y = _data(N, 3, N)
    Xu = np.random.default_rng(N).uniform(-3.6, 3.6, (40, 3))
    k = g.SEIso(0.3, 0.2) + g.LinIso(0.6)                          # a k(x, x) that depends on x: FITC's g term
    _compare(_model(mode, k, X, Xu, y), X, Xu, y, mode, None, "%s N=%d" % (mode, N))


@pytest.mark.parametrize("fast", [True, False])
def test_fsa_block_tile_edges(fast):
    """blocks of 1, 127, 128, 129 and 2048 points; SEIso takes the register path of both contractions, SEIso + LinIso the
    kernel-program path with a non-zero block diagonal"""
    import gpb200 as g
    sizes = (1, 127, 128, 129, 2048)
    N = sum(sizes)
    X, y = _data(N, 3, 17, L=6.0)
    Xu = np.random.default_rng(18).uniform(-5.4, 5.4, (60, 3))
    blocks = _blocks(N, 19, sizes)
    k = g.SEIso(0.3, 0.2) if fast else g.SEIso(0.3, 0.2) + g.LinIso(0.6)
    _compare(_model("FSA", k, X, Xu, y, blocks), X, Xu, y, "FSA", blocks, "FSA blocks %s fast=%s" % (sizes, fast))


@pytest.mark.parametrize("mode", MODES)
def test_invariants(mode):
    import gpb200 as g
    d, N, M = 3, 3000, 128
    X, y = _data(N, d, 5)
    Xu = np.random.default_rng(6).uniform(-3.6, 3.6, (M, d))
    blocks = _blocks(N, 7) if mode == "FSA" else None
    k = g.SEArd([-0.2, 0.0, 0.1], 0.1) + g.RQIso(0.2, -0.3, 0.1)
    gp = _model(mode, k, X, Xu, y, blocks)
    e = gp._eng
    Xs = np.random.default_rng(8).uniform(-4, 4, (200, d))
    r = y - 0.1

    def state():
        a, m, ld = e.mll(r)
        out = [a, np.array([m, ld])]
        if mode == "FSA":
            out += list(e.predict_fsa(Xs, np.full(200, 2, dtype=np.int64)))
        else:
            out += list(e.predict(Xs))
        return out

    s0 = state()
    gk0 = e.grad_kernel()
    _, gu0 = e.grad_kernel_inducing(want_kernel=False)
    gk1, gu1, gx1 = e.grad_kernel_inputs(want_kernel=True, want_inducing=True)
    np.testing.assert_array_equal(gk1, gk0)                    # the kernel and Xu parts are those of the other calls
    np.testing.assert_array_equal(gu1, gu0)
    for a, b in zip(s0, state()):
        np.testing.assert_array_equal(a, b)                    # mll, alpha and predictions are unchanged by the call
    for wk, wu in ((False, False), (True, False), (False, True)):
        gk, gu, gx = e.grad_kernel_inputs(want_kernel=wk, want_inducing=wu)
        np.testing.assert_array_equal(gx, gx1)                 # repeated calls, with and without the other parts
        assert (gk is None) != wk and (gu is None) != wu
    np.testing.assert_array_equal(e.grad_kernel(), gk0)
    t = e.grad_inputs_timings()
    assert 0.0 < t[0] <= t[1], t
    # set_inputs + factorize + mll == a fresh handle given the new X (and the same blocks), bitwise
    X2 = X + 0.05 * np.random.default_rng(9).standard_normal(X.shape)
    p = gp.get_params(inputs=True)
    gp.set_params(np.concatenate([p[:p.size - X.size], X2.ravel()]), inputs=True)
    gp.update_mll()
    fresh = _model(mode, k, X2, Xu, y, blocks)
    np.testing.assert_array_equal(gp.alpha, fresh.alpha)
    assert gp.mll == fresh.mll and gp.logdet == fresh.logdet
    gp.update_dmll(inputs=True, inducing=True)
    fresh.update_dmll(inputs=True, inducing=True)
    np.testing.assert_array_equal(gp.dmll, fresh.dmll)


def test_error_codes():
    import gpb200 as g
    from gpb200 import capi
    X, y = _data(500, 2, 10)
    Xu = X[:20].copy()
    gp = g.FITC(X.T, Xu.T, y, g.MeanZero(), g.SEIso(0.0, 0.0), -1.0)
    lib, h = gp._eng._lib, gp._eng._h
    gx = np.empty((500, 2))
    pd = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    Xc = np.ascontiguousarray(X)
    assert lib.gpb200_fitc_grad_kernel_inputs(h, None, None, None) == capi.EINVAL
    assert lib.gpb200_fitc_set_inputs(h, 499, pd(Xc), 2) == capi.EINVAL
    assert lib.gpb200_fitc_set_inputs(h, 500, None, 2) == capi.EINVAL
    assert lib.gpb200_fitc_set_inputs(h, 500, pd(Xc), 1) == capi.EINVAL
    assert lib.gpb200_fitc_set_inputs(h, 500, pd(Xc), 2) == capi.OK
    assert lib.gpb200_fitc_grad_kernel_inputs(h, None, None, pd(gx)) == capi.ESTATE     # factorize + mll first
    gp.update_mll()
    assert lib.gpb200_fitc_grad_kernel_inputs(h, None, None, pd(gx)) == capi.OK
    e = capi.FitcEngine()
    assert e._lib.gpb200_fitc_set_inputs(e._h, 500, pd(Xc), 2) == capi.ESTATE           # set_data first
    e.set_data(Xc, np.ascontiguousarray(Xu))
    e.set_kernel(*g.kernels.flatten(g.SEIso(0.0, 0.0), 2)[:2], 2)
    with pytest.raises(ValueError):
        e.grad_kernel_inputs()
    with pytest.raises(ValueError):
        e.set_inputs(Xc[:5])
    e.close()


def _directional(gp, D, h):
    """sixth-order central difference of the device mll along D (an (N, d) step of the training inputs)"""
    p = gp.get_params(inputs=True)
    nx = D.size
    f = []
    for s in (-3, -2, -1, 1, 2, 3):
        q = p.copy()
        q[p.size - nx:] += s * h * D.ravel()
        gp.set_params(q, inputs=True)
        gp.update_mll()
        f.append(gp.mll)
    gp.set_params(p, inputs=True)
    gp.update_mll()
    return (-f[0] + 9.0 * f[1] - 45.0 * f[2] + 45.0 * f[3] - 9.0 * f[4] + f[5]) / (60.0 * h)


@pytest.mark.parametrize("mode,N,M,d", [("FITC", 1_000_000, 4096, 8), ("FSA", 200_000, 1024, 3)])
def test_directional_derivative_at_scale(mode, N, M, d):
    import gpb200 as g
    L = 3.0 if d == 8 else 8.0
    X, y = _data(N, d, 11, L=L)
    rng = np.random.default_rng(12)
    Xu = X[rng.permutation(N)[:M]] + 0.01 * rng.standard_normal((M, d))
    blocks = [np.arange(i, min(i + 512, N)) for i in range(0, N, 512)] if mode == "FSA" else None
    gp = _model(mode, g.SEIso(np.log(2.0) if d == 8 else 0.0, 0.0), X, Xu, y, blocks)
    if mode == "FITC":
        assert gp._eng.N > 32768                                      # several staging chunks
    gp.update_dmll(inputs=True)
    gx = gp.dmll[-X.size:].reshape(N, d)
    D = rng.standard_normal((N, d))
    dd = float(np.sum(gx * D))
    fds = [_directional(gp, D, h) for h in (1e-3, 3e-4)]
    fd = min(fds, key=lambda v: abs(v - dd))
    rel = abs(dd - fd) / np.linalg.norm(gx)
    print("%s N=%d M=%d d=%d: <g, D> %.10e  fd %s  |g| %.3e  rel %.2e  timings %s" % (
        mode, N, M, d, dd, fds, np.linalg.norm(gx), rel, gp._eng.grad_inputs_timings()))
    assert rel <= 1e-6


def test_optimize_inputs_and_inducing():
    """perturbed inputs: moving X and Xu together raises the mll above optimising the hyper-parameters alone (the rollback
    of a rejected step is the host's, tests/test_sparse_inputs_host_cpu.py)"""
    import gpb200 as g
    rng = np.random.default_rng(13)
    N, M, d = 1500, 15, 2
    X0 = rng.uniform(-3, 3, (N, d))
    y = np.sin(X0[:, 0]) * np.cos(X0[:, 1]) + 0.05 * rng.standard_normal(N)
    X = X0 + 0.3 * rng.standard_normal((N, d))                      # observed sites, perturbed
    Xu = rng.uniform(-2.5, 2.5, (M, d))
    blocks = [np.arange(i, min(i + 300, N)) for i in range(0, N, 300)]
    mk = lambda: g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.SEIso(np.log(0.7), 0.0), -2.0)
    a, b = mk(), mk()
    ra = a.optimize(maxiter=60)
    rb = b.optimize(inputs=True, inducing=True, maxiter=60)
    print("optimize(): mll %.6f (%d it)   optimize(inputs, inducing): mll %.6f (%d it)" % (a.mll, ra.nit, b.mll, rb.nit))
    assert b.mll > a.mll + 1.0
    np.testing.assert_array_equal(a.x, X.T)                          # optimize() leaves X alone
    np.testing.assert_array_equal(b.get_params(inputs=True, inducing=True), rb.x)


def test_optimize_rolls_back_a_singular_step_on_the_device(monkeypatch):
    """a step that puts two training points of one FSA block on the same site makes that block of Lambda singular: the
    device factorisation reports it (PosDefException) and optimize's exception filter rolls the parameters back, X and Xu
    included.  LinIso with the site (2^20, 0) and the inducing point (0, 1): K_fu is 0 there and K_bb is 2^40 in every
    entry of the pair, which the noise (below half an ulp of 2^40) does not change, so the second pivot is exactly 0."""
    import scipy.optimize
    import gpb200 as g
    from gpb200.capi import PosDefException
    rng = np.random.default_rng(14)
    N, d = 40, 2
    X = rng.standard_normal((N, d))
    y = X[:, 0] + 0.1 * rng.standard_normal(N)
    Xu = np.array([[0.0, 1.0]])
    blocks = [np.arange(i, i + 10) for i in range(0, N, 10)]
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.LinIso(0.0), -6.0)
    flags = dict(inputs=True, inducing=True)
    p0 = gp.get_params(**flags)
    m0, a0 = gp.mll, gp.alpha.copy()
    assert np.isfinite(m0)
    bad = p0.copy()
    nx = X.size
    bad[p0.size - nx:p0.size - nx + 4] = [2.0 ** 20, 0.0, 2.0 ** 20, 0.0]      # x_0 = x_1, both in block 0
    with pytest.raises(PosDefException):
        gp.set_params(bad, **flags)
        gp.update_mll()
    gp.set_params(p0, **flags)
    gp.update_mll()
    assert gp.mll == m0
    seen = []

    def one_bad_step(fun, x0, jac=None, method=None, options=None, **kw):
        """stands in for L-BFGS: the singular point first, then the start; the model's own fg does the rest"""
        f_bad, g_bad = fun(bad)
        seen.append((f_bad, g_bad, gp.get_params(**flags)))
        f0, _ = fun(np.asarray(x0))
        seen.append(f0)
        return scipy.optimize.OptimizeResult(x=np.asarray(x0), nit=1, fun=f0)

    monkeypatch.setattr(scipy.optimize, "minimize", one_bad_step)
    gp.optimize(**flags)
    f_bad, g_bad, p_after = seen[0]
    assert f_bad >= 1e10                                              # the rejected step's penalty
    np.testing.assert_array_equal(g_bad, bad - p0)                    # pointing back to the last accepted point
    np.testing.assert_array_equal(p_after, p0)                        # X and Xu rolled back
    assert seen[1] == -m0
    np.testing.assert_array_equal(gp.get_params(**flags), p0)
    assert gp.mll == m0
    np.testing.assert_array_equal(gp.alpha, a0)
