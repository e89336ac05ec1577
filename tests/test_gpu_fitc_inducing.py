"""GPU: dmll/dXu of FITC, DTC, SoR and FSA (gpb200_fitc_grad_kernel_inducing) against the dense oracle
(inducing_grad_oracle.dmll_dxu) over the kernel zoo and at M below, at and above one 128-tile; the invariants of the joint
call and of gpb200_fitc_set_inducing; directional derivatives at scale against central differences of the device mll;
and optimize(inducing=True) end to end."""
import ctypes as C

import numpy as np
import pytest

from conftest import kernel_zoo
import inducing_grad_oracle as ig

pytestmark = pytest.mark.gpu
MODES = ("FITC", "DTC", "SoR", "FSA")
# the linear-feature kernels have rank d + 1 (LinIso + Const) and 10 (degree-2 Poly at d = 3): more inducing points leave
# K_uu singular up to its nugget; Periodic(1d) sees one coordinate only
M_OF = {"LinIso+Const": 3, "Poly": 6, "Periodic(1d)": 4}


def _blocks(N, seed):
    """a partition of 0..N-1 into blocks of mixed sizes (1, 127, 128, 129, 300, 64, ...): every padding case of the layout"""
    perm = np.random.default_rng(seed).permutation(N)
    sizes, out, i, k = (1, 127, 128, 129, 300, 64), [], 0, 0
    while i < N:
        out.append(np.sort(perm[i:i + sizes[k % len(sizes)]]))
        i += sizes[k % len(sizes)]
        k += 1
    return out


def _model(mode, kernel, X, Xu, y, blocks=None, ln=-1.0):
    import gpb200 as g
    if mode == "FSA":
        return g.FSA(X.T, Xu.T, blocks, y, g.MeanConst(0.1), kernel, ln)
    return getattr(g, mode)(X.T, Xu.T, y, g.MeanConst(0.1), kernel, ln)


def _data(N, d, seed, L=4.0):
    """N points in [-L, L]^d: wide enough against the zoo's length scales that K_uu stays away from singular at M = 300"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-L, L, (N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    return X, y


def _compare(gp, X, Xu, y, mode, blocks, tag):
    spec = gp.kernel.spec()
    _, gx = gp._eng.grad_kernel_inducing(want_kernel=False)
    go = ig.dmll_dxu(spec, X, Xu, y, gp.logNoise, mode, blocks, mspec=("MeanConst", 0.1))
    c_uu, c_s = ig.conditioning(spec, X, Xu, gp.logNoise, mode, blocks)
    err = np.max(np.abs(gx - go))
    scale = np.max(np.abs(go))
    print("%-40s cond(K_uu) %.2e cond(S_QR) %.2e  max|err| %.3e  max|g| %.3e  rel %.2e" % (tag, c_uu, c_s, err, scale, err / scale))
    # the kernel gradient's bound (rtol 1e-6, atol 1e-7), taken against the largest entry: every entry is a sum over the
    # same adjoints, so the small ones carry the large ones' absolute error
    assert err <= 1e-6 * scale + 1e-7, tag
    # and a bound in the conditioning: both gradients go through Sigma_QR^-1 (the device's explicit inverse, the oracle's
    # dense S^-1), and the error follows cond(Sigma_QR) rather than cond(K_uu)
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
@pytest.mark.parametrize("case", ["SEIso", "Mat32Ard", "Mat12Iso, Xu in x", "SE*RQ, Xu in x"])
def test_sizes_parity(mode, N, M, case):
    d = 3
    X, y = _data(N, d, N + M, L=7.0)
    name = case.split(",")[0]
    rng = np.random.default_rng(M)
    Xu = X[rng.permutation(N)[:M]].copy() if "Xu in x" in case else rng.uniform(-6.3, 6.3, (M, d))
    blocks = _blocks(N, 4) if mode == "FSA" else None
    gp = _model(mode, dict(kernel_zoo(d))[name], X, Xu, y, blocks)
    _compare(gp, X, Xu, y, mode, blocks, "%s %s N=%d M=%d" % (mode, case, N, M))


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
        out = [a, np.array([m, ld]), e.grad_kernel()]
        if mode == "FSA":
            out += list(e.predict_fsa(Xs, np.full(200, 2, dtype=np.int64)))
        else:
            out += list(e.predict(Xs)) + list(e.cv_param(0))
        return out

    s0 = state()
    gk0 = e.grad_kernel()
    gk1, gx1 = e.grad_kernel_inducing()
    np.testing.assert_array_equal(gk1, gk0)                    # the joint call's kernel part is grad_kernel's, bitwise
    s1 = state()
    for a, b in zip(s0, s1):
        np.testing.assert_array_equal(a, b)                    # an intervening joint call changes nothing else
    _, gx2 = e.grad_kernel_inducing(want_kernel=False)
    gk3, gx3 = e.grad_kernel_inducing()
    np.testing.assert_array_equal(gx2, gx1)                    # repeated calls, with and without the kernel part
    np.testing.assert_array_equal(gx3, gx1)
    np.testing.assert_array_equal(gk3, gk0)
    t = e.grad_inducing_timings()
    assert 0.0 < t[0] <= t[1], t
    # set_inducing + factorize + mll == a fresh handle given the new Xu, bitwise
    Xu2 = Xu + 0.05 * np.random.default_rng(9).standard_normal(Xu.shape)
    p = gp.get_params(inducing=True)
    gp.set_params(np.concatenate([p[:p.size - Xu.size], Xu2.ravel()]), inducing=True)
    gp.update_mll()
    fresh = _model(mode, k, X, Xu2, y, blocks)
    np.testing.assert_array_equal(gp.alpha, fresh.alpha)
    assert gp.mll == fresh.mll and gp.logdet == fresh.logdet
    gp.update_dmll(inducing=True)
    fresh.update_dmll(inducing=True)
    np.testing.assert_array_equal(gp.dmll, fresh.dmll)


def test_error_codes():
    import gpb200 as g
    from gpb200 import capi
    X, y = _data(500, 2, 10)
    Xu = X[:20].copy()
    gp = g.FITC(X.T, Xu.T, y, g.MeanZero(), g.SEIso(0.0, 0.0), -1.0)
    lib, h = gp._eng._lib, gp._eng._h
    gx = np.empty((20, 2))
    pd = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    assert lib.gpb200_fitc_grad_kernel_inducing(h, None, None) == capi.EINVAL
    assert lib.gpb200_fitc_set_inducing(h, 19, pd(Xu), 2) == capi.EINVAL
    assert lib.gpb200_fitc_set_inducing(h, 20, None, 2) == capi.EINVAL
    assert lib.gpb200_fitc_set_inducing(h, 20, pd(Xu), 1) == capi.EINVAL
    assert lib.gpb200_fitc_set_inducing(h, 20, pd(np.ascontiguousarray(Xu)), 2) == capi.OK
    assert lib.gpb200_fitc_grad_kernel_inducing(h, None, pd(gx)) == capi.ESTATE      # factorize + mll first
    gp.update_mll()
    assert lib.gpb200_fitc_grad_kernel_inducing(h, None, pd(gx)) == capi.OK
    e = capi.FitcEngine()
    assert e._lib.gpb200_fitc_set_inducing(e._h, 20, pd(Xu), 2) == capi.ESTATE        # set_data first
    e.set_data(np.ascontiguousarray(X), np.ascontiguousarray(Xu))
    e.set_kernel(*g.kernels.flatten(g.SEIso(0.0, 0.0), 2)[:2], 2)
    with pytest.raises(ValueError):
        e.grad_kernel_inducing()
    with pytest.raises(ValueError):
        e.set_inducing(Xu[:5])
    e.close()


def _directional(gp, D, h):
    """sixth-order central difference of the device mll along D (an (M, d) step of the inducing points)"""
    p = gp.get_params(inducing=True)
    nu = D.size
    f = []
    for s in (-3, -2, -1, 1, 2, 3):
        q = p.copy()
        q[p.size - nu:] += s * h * D.ravel()
        gp.set_params(q, inducing=True)
        gp.update_mll()
        f.append(gp.mll)
    gp.set_params(p, inducing=True)
    gp.update_mll()
    return (-f[0] + 9.0 * f[1] - 45.0 * f[2] + 45.0 * f[3] - 9.0 * f[4] + f[5]) / (60.0 * h)


@pytest.mark.parametrize("mode,N,M", [("FITC", 1_000_000, 4096), ("FSA", 200_000, 1024)])
def test_directional_derivative_at_scale(mode, N, M):
    import gpb200 as g
    d = 3
    X, y = _data(N, d, 11, L=12.0 if mode == "FITC" else 8.0)    # about 1.5 length scales between inducing points
    rng = np.random.default_rng(12)
    Xu = X[rng.permutation(N)[:M]] + 0.01 * rng.standard_normal((M, d))
    blocks = [np.arange(i, min(i + 512, N)) for i in range(0, N, 512)] if mode == "FSA" else None
    gp = _model(mode, g.SEIso(0.0, 0.0), X, Xu, y, blocks)
    if mode == "FITC":
        assert gp._eng.N > 32768                                      # several staging chunks
    gp.update_dmll(inducing=True)
    gx = gp.dmll[-Xu.size:].reshape(M, d)
    D = rng.standard_normal((M, d))
    dd = float(np.sum(gx * D))
    fds = [_directional(gp, D, h) for h in (1e-3, 3e-4)]
    fd = min(fds, key=lambda v: abs(v - dd))
    # a standard-normal D makes <g, D> of the size of |g|, which the tolerance is relative to
    rel = abs(dd - fd) / np.linalg.norm(gx)
    print("%s N=%d M=%d: <g, D> %.10e  fd %s  |g| %.3e  rel %.2e  timings %s" % (mode, N, M, dd, fds, np.linalg.norm(gx), rel,
                                                                                  gp._eng.grad_inducing_timings()))
    # the rounding of the device mll, divided by the step, limits the difference quotient at N = 10^6: the closer of two
    # steps is kept
    assert rel <= 1e-6


def test_optimize_moves_bunched_inducing_points():
    import gpb200 as g
    rng = np.random.default_rng(13)
    N, M, d = 2000, 20, 2
    X = rng.uniform(-3, 3, (N, d)); y = np.sin(X[:, 0]) * np.cos(X[:, 1]) + 0.1 * rng.standard_normal(N)
    gx, gy = np.meshgrid(np.linspace(1.5, 2.9, 5), np.linspace(2.0, 2.9, 4))
    Xu = np.c_[gx.ravel(), gy.ravel()]                                    # all in one corner of [-3, 3]^2
    a = g.FITC(X.T, Xu.T, y, g.MeanZero(), g.SEIso(np.log(0.5), 0.0), -1.0)
    b = g.FITC(X.T, Xu.T, y, g.MeanZero(), g.SEIso(np.log(0.5), 0.0), -1.0)
    ra = a.optimize(maxiter=100)
    rb = b.optimize(inducing=True, maxiter=100)
    moved = np.max(np.linalg.norm(b.Xu - Xu.T, axis=0))
    print("optimize(): mll %.6f (%d it)   optimize(inducing=True): mll %.6f (%d it), largest move %.3f" % (a.mll, ra.nit, b.mll, rb.nit, moved))
    assert b.mll > a.mll + 1.0
    assert moved > 0.5
    np.testing.assert_array_equal(a.Xu, Xu.T)                              # optimize() leaves Xu alone
    np.testing.assert_array_equal(b.get_params(inducing=True), rb.x)
    c = g.FITC(X.T, b.Xu, y, g.MeanZero(), g.SEIso(np.log(0.5), 0.0), -1.0)   # the final state is an ordinary model
    c.set_params(rb.x, inducing=True)
    c.update_mll()
    assert c.mll == b.mll
