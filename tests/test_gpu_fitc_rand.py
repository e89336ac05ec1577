"""GPU: posterior draws of the sparse strategies (rand(gp, X, n), src/GP.jl:120-146, with cK a FITC / DTC / SoR / FSA
covariance) and the GPE parameter protocol on them (get_params / set_params / update_target* / optimize, src/GPE.jl:346-510,
src/optimize.jl).

Parity.  With the same standard-normal draws Z the samples are mu* + chol(Sigma* + nugget I) Z.  The device's Sigma* is the
covariance predict_f(full_cov=true) returns (the engine builds it with the same code), so the draws are checked at 1e-8
against numpy's Cholesky of that matrix -- this isolates make_posdef!, the Cholesky and unwhiten! -- and Sigma* itself against
the oracle at the full-covariance tolerance of test_gpu_fitc.py / test_gpu_fsa.py, and the draws against the oracle's at
max(1e-8, 64 cond(K_uu) eps) max|want|.  The inducing points lie on a grid (cond(K_uu) ~ 10^2): with random ones the oracle
comparison only bounds conditioning (see test_gpu_fitc.py).  nugget = 1e-6 as in test_gpu_parity.py: SoR's Sigma* has rank <= M < Ms, and the nugget
bounds how much the Cholesky amplifies last-bit differences.

FSA draws pair all test points with one training block.  predictMVN (full_scale_approximation.jl:413-447) takes the exact K**
between test points but Lambda_xf only on the paired block, so test points spread over several test blocks give an indefinite
Sigma* (eigenvalues near -1 here): rand then raises PosDefException, on the device as in the reference."""
import ctypes as C

import numpy as np
import pytest

from oracle import gp_oracle as orc
from fsa_oracle import fsa_fit, fsa_predict_closed, fsa_predict_full

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
NUGGET = 1e-6
MODES = ["FITC", "DTC", "SoR", "FSA"]


def _kernel(g, kname):
    if kname == "SEIso":
        return g.SEIso(-0.3, 0.1)
    if kname == "fixed":
        return g.SEIso(-0.3, 0.1) * g.fix(g.Mat32Iso(0.2, -0.2), "lσ")
    return g.SEIso(-0.3, 0.1) * g.Mat32Iso(0.2, -0.2) + g.Mat12Iso(0.5, -1.5)


def _problem(mode, kname, N=2000, seed=0, ln=-1.0):
    """GP on N points in [-3, 3]^2 with 49 inducing points on a grid; FSA: five training blocks along x_0"""
    import gpb200 as g
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (N, 2)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-2.5, 2.5, 7)
    Xu = np.array([[a, b] for a in grid for b in grid])
    k = _kernel(g, kname)
    blocks = None
    if mode == "FSA":
        order = np.argsort(X[:, 0])
        blocks = [np.sort(order[i:i + N // 5]) for i in range(0, N, N // 5)]
        gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanConst(0.1), k, ln)
    else:
        gp = getattr(g, mode)(X.T, Xu.T, y, g.MeanConst(0.1), k, ln)
    return gp, X, Xu, y, blocks


def _test_points(X, blocks, Ms, seed):
    """Ms test points; FSA: all of them in the x_0 range of training block 2 and paired with it"""
    rng = np.random.default_rng(seed)
    if blocks is None:
        return rng.uniform(-3.5, 3.5, (Ms, 2)), None
    lo, hi = X[blocks[2], 0].min(), X[blocks[2], 0].max()
    none = np.zeros(0, dtype=np.int64)
    return np.c_[rng.uniform(lo, hi, Ms), rng.uniform(-3.5, 3.5, Ms)], [none, none, np.arange(Ms)]


def _cond_kuu(spec, Xu):
    w = np.linalg.eigvalsh(orc.cov(spec, Xu) + 1e-10 * np.eye(Xu.shape[0]))
    return float(w[-1] / w[0])


def _rand(gp, Xs, bpred, n, nugget, rng):
    return gp.rand(Xs.T, bpred, n=n, nugget=nugget, rng=rng) if bpred is not None else gp.rand(Xs.T, n=n, nugget=nugget, rng=rng)


def _predict_full(gp, Xs, bpred):
    return gp.predict_f(Xs.T, bpred, full_cov=True) if bpred is not None else gp.predict_f(Xs.T, full_cov=True)


@pytest.mark.parametrize("Ms", [37, 300, 1000])
@pytest.mark.parametrize("kname", ["SEIso", "composite"])
@pytest.mark.parametrize("mode", MODES)
def test_rand_matches_cholesky_of_the_predictive_covariance(mode, kname, Ms):
    gp, X, Xu, y, blocks = _problem(mode, kname)
    Xs, bpred = _test_points(X, blocks, Ms, seed=Ms)
    n = 5
    draws = _rand(gp, Xs, bpred, n, NUGGET, np.random.default_rng(1))
    z = np.random.default_rng(1).standard_normal((n, Ms))                   # the draws rand took from the same generator
    assert draws.shape == (Ms, n)
    mu, S = _predict_full(gp, Xs, bpred)
    want = mu[None, :] + z @ np.linalg.cholesky(S + NUGGET * np.eye(Ms)).T
    scale = float(np.max(np.abs(want)))
    e_dev = float(np.max(np.abs(draws.T - want)))
    # Sigma* and the draws against the oracle: 1e-8 max|want|, widened by cond(K_uu) as in test_gpu_fitc.py
    spec, mspec = gp.kernel.spec(), ("MeanConst", 0.1)
    cond = _cond_kuu(spec, Xu)
    tol = max(1e-10, 64.0 * cond * EPS)
    tol_draw = max(1e-8, 64.0 * cond * EPS)
    if mode == "FSA":
        o = fsa_fit(spec, X, Xu, blocks, y, -1.0, mspec)
        mo, So = fsa_predict_closed(spec, X, Xu, o, Xs, bpred, mspec)              # the closed form the device evaluates
        ml, Sl = fsa_predict_full(spec, X, Xu, o, Xs, bpred, mspec)
        assert float(np.max(np.abs(S - Sl))) <= 1e-6 * float(np.max(np.abs(Sl)))     # the literal predictMVN, as test_gpu_fsa.py
        # draws from the literal predictMVN: its Sigma* differs by Sigma_QR's second 1e-10 nugget (test_gpu_fsa.py), which
        # the Cholesky carries at most as |dL|_F <= |L|_2 |dSigma|_F / lambda_min (first order)
        lam = np.linalg.eigvalsh(Sl + NUGGET * np.eye(Ms))
        dL = np.sqrt(lam[-1]) * np.linalg.norm(S - Sl) / lam[0]
        bound_l = tol_draw * scale + float(np.max(np.abs(mu - ml))) + 2.0 * dL * float(np.max(np.linalg.norm(z, axis=1)))
        e_l = float(np.max(np.abs(draws.T - (ml[None, :] + z @ np.linalg.cholesky(Sl + NUGGET * np.eye(Ms)).T))))
        print("    vs the literal FSA predictMVN %.2e (first-order bound %.1e)" % (e_l, bound_l))
        assert e_l <= bound_l
    else:
        o = orc.fitc_fit(spec, X, Xu, y, -1.0, mspec, mode=mode)
        mo, So = orc.fitc_predict_full(spec, X, Xu, o, Xs, mspec)
    assert float(np.max(np.abs(S - So))) <= tol * float(np.max(np.abs(So)))
    e_o = float(np.max(np.abs(draws.T - (mo[None, :] + z @ np.linalg.cholesky(So + NUGGET * np.eye(Ms)).T))))
    print("rand %s %s Ms=%d: cond(K_uu)=%.1e  vs chol(device Sigma*) %.2e  vs oracle %.2e  (bounds %.1e / %.1e)"
          % (mode, kname, Ms, cond, e_dev, e_o, 1e-8 * scale, tol_draw * scale))
    assert e_dev <= 1e-8 * scale
    assert e_o <= tol_draw * scale


@pytest.mark.parametrize("mode", MODES)
def test_rand_engine_mean_and_repeatability(mode):
    """The engine's mu is predict's, bitwise; two calls with the same Z return the same draws, bitwise."""
    gp, X, Xu, y, blocks = _problem(mode, "SEIso")
    Xs, bpred = _test_points(X, blocks, 200, seed=3)
    from gpb200.sparse import test_block_of
    block_of = test_block_of(bpred, 200) if bpred is not None else None
    z = np.random.default_rng(4).standard_normal((7, 200))
    e = gp._eng
    mu1, d1 = e.rand(Xs, z, nugget=1e-8, block_of=block_of)
    mu2, d2 = e.rand(Xs, z, nugget=1e-8, block_of=block_of)
    mp, _ = e.predict_fsa(Xs, block_of, full_cov=True) if mode == "FSA" else e.predict_cov(Xs)
    assert np.array_equal(mu1, mp) and np.array_equal(mu2, mp) and np.array_equal(d1, d2)
    t = e.rand_timings()
    assert t.shape == (3,) and np.all(t > 0.0)


@pytest.mark.parametrize("mode", MODES)
def test_rand_mean_of_many_draws(mode):
    """The mean of 70 000 draws (more than gridDim.y allows in one launch) lies within 5 sigma / sqrt(n) of predict_f
    (sigma^2 = the predictive variance + nugget)."""
    gp, X, Xu, y, blocks = _problem(mode, "composite")
    Xs, bpred = _test_points(X, blocks, 50, seed=5)
    n, nugget = 70000, 1e-8
    draws = _rand(gp, Xs, bpred, n, nugget, np.random.default_rng(6))
    mu, var = gp.predict_f(Xs.T, bpred) if bpred is not None else gp.predict_f(Xs.T)
    dev = np.abs(draws.mean(axis=1) - mu)
    sd = np.sqrt((var + nugget) / n)
    assert np.all(dev <= 5.0 * sd), np.max(dev / sd)


def _raw(e, Ms, xs, ldxs, block_of, nsamp, z, nugget, mu, out):
    lp = C.POINTER(C.c_int64)
    dp = C.POINTER(C.c_double)
    as_dp = lambda a: a.ctypes.data_as(dp) if a is not None else None
    return e._lib.gpb200_fitc_rand(e._h, Ms, as_dp(xs), ldxs, block_of.ctypes.data_as(lp) if block_of is not None else None,
                                   nsamp, as_dp(z), nugget, as_dp(mu), as_dp(out))


def test_rand_error_codes():
    import gpb200 as g
    from gpb200 import capi
    rng = np.random.default_rng(7)
    X = rng.uniform(-3, 3, (1000, 2)); Xu = X[:30]
    ops, dims, theta, _ = g.flatten(g.SEIso(-0.3, 0.1), 2)
    Ms = 40
    xs = np.ascontiguousarray(rng.uniform(-3, 3, (Ms, 2)))
    z = rng.standard_normal((3, Ms)); mu = np.empty(Ms); out = np.empty((3, Ms))
    e = capi.FitcEngine(0)
    e.set_data(X, Xu)
    e.set_kernel(ops, dims, theta.size)
    assert _raw(e, Ms, xs, 2, None, 3, z, 1e-10, mu, out) == capi.ESTATE               # before factorize
    e.factorize(theta, -1.0)
    assert _raw(e, Ms, xs, 2, None, 3, z, 1e-10, mu, out) == capi.ESTATE               # before mll
    e.mll(np.sin(X.sum(1)))
    assert _raw(e, Ms, xs, 2, None, 3, z, 1e-10, mu, out) == capi.OK
    block_of = np.zeros(Ms, dtype=np.int64)
    bad = [(0, xs, 2, None, 3, z, 1e-10, mu, out), (Ms, xs, 2, None, 0, z, 1e-10, mu, out), (Ms, xs, 1, None, 3, z, 1e-10, mu, out),
           (Ms, None, 2, None, 3, z, 1e-10, mu, out), (Ms, xs, 2, None, 3, None, 1e-10, mu, out),
           (Ms, xs, 2, None, 3, z, 1e-10, None, out), (Ms, xs, 2, None, 3, z, 1e-10, mu, None),
           (Ms, xs, 2, None, 3, z, -1e-12, mu, out), (Ms, xs, 2, None, 3, z, float("nan"), mu, out),
           (Ms, xs, 2, block_of, 3, z, 1e-10, mu, out)]                                   # block_of outside FSA mode
    for args in bad:
        assert _raw(e, *args) == capi.EINVAL, args
    big = np.ascontiguousarray(rng.uniform(-3, 3, (1025, 2)))                            # one staging chunk holds 1024 rows here
    zb = rng.standard_normal((2, 1025))
    assert _raw(e, 1025, big, 2, None, 2, zb, 1e-10, np.empty(1025), np.empty((2, 1025))) == capi.EINVAL
    assert _raw(e, Ms, xs, 2, None, 3, z, 1e-10, mu, out) == capi.OK                     # the handle is still usable
    e.close()
    # FSA: block_of is required, too many padded test rows is EINVAL
    gp, X, Xu, y, blocks = _problem("FSA", "SEIso", N=1000)
    Xs, bpred = _test_points(X, blocks, Ms, seed=8)
    xs = np.ascontiguousarray(Xs)
    assert _raw(gp._eng, Ms, xs, 2, None, 3, z, 1e-10, mu, out) == capi.EINVAL
    assert _raw(gp._eng, Ms, xs, 2, block_of + 2, 3, z, 1e-8, mu, out) == capi.OK
    Mbig = 40000
    xb = np.ascontiguousarray(np.random.default_rng(9).uniform(-3, 3, (Mbig, 2)))
    zb = np.zeros((1, Mbig))
    assert _raw(gp._eng, Mbig, xb, 2, np.zeros(Mbig, dtype=np.int64), 1, zb, 1e-10, np.empty(Mbig), np.empty((1, Mbig))) == capi.EINVAL
    with pytest.raises(TypeError):
        gp.rand(Xs.T)
    with pytest.raises(ValueError, match="two prediction blocks"):
        gp.rand(Xs.T, [[0, 1], [1, 2]])


def test_rand_not_positive_definite_raises_and_the_handle_stays_usable():
    """SoR, test points so far from every inducing point that K_*u underflows to 0: Sigma* = 0 and with nugget 0 the first
    pivot fails.  PosDefException; afterwards the same handle draws again, bitwise as before."""
    import gpb200 as g
    gp, X, Xu, y, blocks = _problem("SoR", "SEIso")
    Xs, _ = _test_points(X, None, 60, seed=10)
    before = gp.rand(Xs.T, n=4, nugget=1e-8, rng=np.random.default_rng(11))
    far = Xs + 1e3
    with pytest.raises(g.PosDefException) as ex:
        gp.rand(far.T, n=4, nugget=0.0, rng=np.random.default_rng(11))
    print("far test points: PosDefException(%d)" % ex.value.info)
    assert ex.value.info >= 1
    after = gp.rand(Xs.T, n=4, nugget=1e-8, rng=np.random.default_rng(11))
    assert np.array_equal(before, after)
    far_ok = gp.rand(far.T, n=2, nugget=1e-6, rng=np.random.default_rng(12))          # Sigma* = 0 + nugget: mean + 1e-3 z
    assert np.allclose(far_ok, 0.1, atol=1e-2)


def test_fsa_rand_over_several_test_blocks_is_not_positive_definite():
    """Test points spread over the five test blocks: Sigma* is indefinite (see the module docstring) -> PosDefException; the
    handle still draws for one test block afterwards."""
    import gpb200 as g
    gp, X, Xu, y, blocks = _problem("FSA", "SEIso")
    Xs = np.random.default_rng(21).uniform(-3, 3, (37, 2))
    edges = [X[b, 0].max() for b in blocks]
    j = np.minimum(np.searchsorted(edges, Xs[:, 0]), len(blocks) - 1)
    bpred = [np.flatnonzero(j == b) for b in range(len(blocks))]
    S = gp.predict_f(Xs.T, bpred, full_cov=True)[1]
    print("FSA Sigma* over %d test blocks: min eigenvalue %.3e" % (sum(b.size > 0 for b in bpred), np.linalg.eigvalsh(S)[0]))
    with pytest.raises(g.PosDefException):
        gp.rand(Xs.T, bpred, n=2, nugget=1e-6, rng=np.random.default_rng(22))
    Xs1, bp1 = _test_points(X, blocks, 37, seed=23)
    assert gp.rand(Xs1.T, bp1, n=2, nugget=1e-6, rng=np.random.default_rng(22)).shape == (37, 2)


@pytest.mark.parametrize("mode", MODES)
def test_rand_leaves_the_handle_state_bitwise_unchanged(mode):
    gp, X, Xu, y, blocks = _problem(mode, "composite")
    Xs, bpred = _test_points(X, blocks, 120, seed=13)
    e = gp._eng

    def state():
        alpha, mll, logdet = e.mll(gp.y - gp.mean.mean(gp._xpm))
        out = [alpha, np.array([mll, logdet, e.grad_noise()]), e.grad_kernel()]
        from gpb200.sparse import test_block_of
        if mode == "FSA":
            out.extend(e.predict_fsa(Xs, test_block_of(bpred, Xs.shape[0])))
        else:
            out.extend(e.predict(Xs))
            out.extend(e.cv_param(0))
            out.append(e.inverse_diag())
        return out

    s0 = state()
    _rand(gp, Xs, bpred, 3, 1e-8, np.random.default_rng(14))
    s1 = state()
    _rand(gp, Xs[:50], [b[b < 50] for b in bpred] if bpred is not None else None, 2, 1e-8, np.random.default_rng(15))
    s2 = state()
    for a, b, c in zip(s0, s1, s2):
        assert np.array_equal(a, b) and np.array_equal(a, c)


def _fd(gp, h):
    p0 = gp.get_params()
    out = []
    for i in range(p0.size):
        vals = []
        for sgn in (1, -1):
            q = p0.copy(); q[i] += sgn * h
            gp.set_params(q)
            gp.update_target()
            vals.append(gp.target)
        out.append((vals[0] - vals[1]) / (2 * h))
    gp.set_params(p0)
    gp.update_target()
    return np.array(out)


@pytest.mark.parametrize("mode", MODES)
def test_dtarget_matches_finite_differences_through_set_params(mode):
    """test/test_sparse.jl:137-141 on the device: central differences of target through set_params against dtarget, over
    [logNoise; mean; kernel] (the FixedKernel parameter is neither exposed nor differentiated)."""
    gp, X, Xu, y, blocks = _problem(mode, "fixed", N=3000, seed=19)
    assert gp.num_params() == 1 + 1 + 3
    gp.update_target_and_dtarget()
    fd = _fd(gp, 1e-4)
    print("%s dtarget %s\n    central differences %s" % (mode, gp.dtarget, fd))
    assert gp.dtarget.shape == fd.shape
    assert np.all(np.abs(gp.dtarget - fd) <= 1e-5 * np.abs(fd) + 1e-4), (gp.dtarget, fd)        # as test_gpu_fitc.py


@pytest.mark.parametrize("mode", MODES)
def test_optimize_raises_the_target(mode):
    gp, X, Xu, y, blocks = _problem(mode, "SEIso", N=1500, seed=20, ln=0.5)
    gp.kernel.set_params([1.0, -1.0])
    gp.initialise_target()
    t0 = gp.target
    ln0 = gp.logNoise
    res = gp.optimize(noise=False, maxiter=15)
    assert gp.logNoise == ln0 and gp.target > t0, (gp.target, t0, res)
    t1 = gp.target
    gp.optimize(maxiter=15)
    assert gp.target > t1 and gp.logNoise != ln0
    p = gp.get_params()
    gp.update_target()
    assert np.array_equal(gp.get_params(), p)
