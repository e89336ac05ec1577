"""GPU parity tests proper: the CUDA path, called through the C ABI (ctypes -> libgpb200.so), against
the CPU oracle on identical (x, y, hyper-parameters).

Tolerances (north-star): 1e-10 relative on log-mll, alpha (normwise: max|Δ| / max|alpha|),
predictive mean and variance; 1e-8 relative on dmll.  All FP64."""
import os

import numpy as np
import pytest

from oracle import gp_oracle as orc
from conftest import make_data, kernel_zoo

pytestmark = pytest.mark.gpu

RTOL = 1e-10
GTOL = 1e-8


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _setup(engine, kernel, X, nb=None, gemm=None):
    import gpb200
    engine.set_data(X)
    ops, dims, theta, exposed = gpb200.flatten(kernel, X.shape[1])
    engine.set_kernel(ops, dims, theta.size)
    if nb is not None:
        engine.set_option("nb", nb)
    if gemm is not None:
        engine.set_option("gemm", gemm)
    return theta, exposed


@pytest.mark.parametrize("idx", range(20))
def test_gram_matches_oracle(engine, idx):
    """cov! parity (kernels.jl:39-50) incl. noise on the diagonal, N not a multiple of the tile."""
    d = 3
    X, y, _ = make_data(300, d, 21)
    name, k = kernel_zoo(d)[idx]
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    ln = -0.5
    try:
        engine.factorize(theta, ln)
    except np.linalg.LinAlgError:
        pass                                    # Gram parity does not need a PD matrix
    K = engine.gram()
    Ko = orc.gram(k.spec(), X, ln)
    assert _rel(K, Ko) < 1e-14, name
    assert np.array_equal(K, K.T)


@pytest.mark.parametrize("idx", range(20))
def test_mll_grad_predict_match_oracle_kernel_zoo(engine, idx):
    d = 3
    X, y, Xs = make_data(300, d, 22, m=37)
    name, k = kernel_zoo(d)[idx]
    theta, exposed = _setup(engine, k, X, nb=256, gemm=0)
    ln = -0.4
    mspec = ("MeanConst", 0.3)
    o = orc.mll_and_dmll(k.spec(), X, y, ln, mspec)
    engine.factorize(theta, ln)
    alpha, mll = engine.mll(y - 0.3)
    assert abs(mll - o["mll"]) <= RTOL * abs(o["mll"]), name
    assert _rel(alpha, o["alpha"]) < RTOL, name
    assert abs(engine.logdet() - o["logdet"]) <= RTOL * abs(o["logdet"]) + 1e-12
    U = engine.factor_upper()
    assert _rel(U, o["U"]) < 1e-11, name
    engine.grad_prepare()
    Kinv = engine.inverse()
    assert _rel(Kinv, np.linalg.inv(o["Ky"])) < 1e-9, name
    gk, trA = engine.grad_kernel()
    assert _rel(gk[exposed], o["dmll_kernel"]) < GTOL, (name, gk[exposed], o["dmll_kernel"])
    assert abs(trA - o["trA"]) <= GTOL * abs(o["trA"]) + 1e-10
    # predict after grad: the factor must still be valid
    mu, var, _ = engine.predict(Xs)
    mo, vo = orc.predict_f(k.spec(), X, o, Xs, ("MeanZero",))
    assert _rel(mu, mo) < RTOL, name
    assert np.max(np.abs(var - vo)) <= RTOL * np.max(np.abs(vo)) + 1e-13, name
    mu2, _, cov = engine.predict(Xs, want_var=False, full_cov=True)
    _, co = orc.predict_f(k.spec(), X, o, Xs, ("MeanZero",), full_cov=True)
    assert _rel(cov, co) < 1e-9, name
    assert np.allclose(cov, cov.T, rtol=0, atol=1e-12)


@pytest.mark.parametrize("N,nb", [(128, 512), (129, 128), (640, 128), (640, 256), (1100, 512), (1537, 256), (2500, 1024), (1100, 0), (2500, 0), (3000, 2048)])
@pytest.mark.parametrize("gemm", [0, 1])
def test_blocking_and_padding(engine, N, nb, gemm):
    """Every recursion shape of the blocked Cholesky / level-parallel inverse, both GEMM loaders."""
    import gpb200
    X, y, Xs = make_data(N, 4, N + nb, m=130)
    k = gpb200.SEIso(0.4, 0.1)
    theta, exposed = _setup(engine, k, X, nb=nb, gemm=gemm)
    ln = -0.6
    o = orc.mll_and_dmll(k.spec(), X, y, ln)
    engine.factorize(theta, ln)
    alpha, mll = engine.mll(y)
    assert abs(mll - o["mll"]) <= RTOL * abs(o["mll"])
    assert _rel(alpha, o["alpha"]) < RTOL
    engine.grad_prepare()
    gk, trA = engine.grad_kernel()
    assert _rel(gk, o["dmll_kernel"]) < GTOL
    assert abs(trA - o["trA"]) <= GTOL * abs(o["trA"])
    assert _rel(engine.solve(y), o["alpha"]) < RTOL
    mu, var, _ = engine.predict(Xs)
    mo, vo = orc.predict_f(k.spec(), X, o, Xs)
    assert _rel(mu, mo) < RTOL
    assert np.max(np.abs(var - vo)) <= RTOL * np.max(np.abs(vo)) + 1e-13
    engine.set_option("gemm", 0)
    engine.set_option("nb", 0)


def test_known_answer_simdata(engine):
    """The reference's own recorded run (perf/benchmarks/simdata.csv, benchmark_julia.ipynb cell 6)."""
    import gpb200
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "simdata_kat.npz"))
    X, Y = np.ascontiguousarray(d["X"]), d["Y"]
    gp = gpb200.GPE(X.T, Y, gpb200.MeanConst(0.0), gpb200.SEIso(0.0, 0.0), 0.0, engine=engine)
    gp.update_target_and_dtarget()
    # current-source semantics (no jitter): SURVEY.md Appendix D2
    assert abs(gp.mll - (-4536.25646128023)) < 1e-10 * 4536.0
    ref = np.array([-689.6318902132696, -15.731253155037956, 71.19489031472071, -667.2676571953316])
    assert np.allclose(gp.dmll, ref, rtol=1e-8)
    assert abs(np.abs(gp.alpha).sum() - 1344.600310514208) < 1e-7
    # historical run: +1e-5 jitter reproduces the recorded mll to 1e-10
    th = np.array([0.0, 0.0])
    engine.factorize(th, 0.0, extra_nugget=1e-5)
    _, mll = engine.mll(Y)
    assert abs(mll - float(d["recorded_mll"])) < 1e-10 * 4536.0
    # benchmark hyper-parameters + predictions: Appendix D3
    gp = gpb200.GPE(X.T, Y, gpb200.MeanConst(0.0), gpb200.SEIso(0.3, 0.3), 0.3, engine=engine)
    gp.update_target_and_dtarget()
    assert abs(gp.mll - (-4955.488218637778)) < 1e-10 * 4955.0
    ref3 = np.array([-1182.9616810127793, -3.211171983399545, 479.3101304593023, -740.5804238604128])
    assert np.allclose(gp.dmll, ref3, rtol=1e-8)
    mu, s2 = gp.predict_f((X[:4] + 0.1).T)
    assert np.allclose(mu, [-0.18841532, -0.34876141, 0.16691408, 0.73227626], atol=2e-8)
    assert np.allclose(s2, [0.75560664, 0.48334666, 0.68344073, 0.6690584], atol=2e-8)


def test_not_positive_definite_is_recoverable(engine):
    """cholesky! throws PosDefException (GP.jl:110); the handle stays usable (optimize.jl:46-61)."""
    import gpb200
    X, y, _ = make_data(260, 2, 3)
    X[200] = X[10]                                   # duplicate point, ~zero noise -> singular K_y
    X[201] = X[10]
    k = gpb200.SEIso(1.0, 0.0)
    theta, _ = _setup(engine, k, X)
    with pytest.raises(gpb200.PosDefException) as ei:
        engine.factorize(theta, -30.0)
    assert 1 <= ei.value.info <= 260
    with pytest.raises(ValueError):
        engine.mll(y)                                # state error: not factorised
    engine.factorize(theta, -1.0)                    # same handle, sane noise
    o = orc.fit(k.spec(), X, y, -1.0)
    alpha, mll = engine.mll(y)
    assert abs(mll - o["mll"]) <= RTOL * abs(o["mll"])


def test_heteroscedastic_noise_vector(engine):
    """logNoise::Vector path of update_cK! (GPE.jl:177-186; test/heteroscedastic.jl)."""
    import gpb200
    X, y, _ = make_data(333, 2, 8)
    ln = -1.0 + 0.5 * np.cos(np.arange(333))
    k = gpb200.Mat52Iso(0.2, 0.1)
    theta, _ = _setup(engine, k, X)
    engine.factorize(theta, ln)
    o = orc.fit(k.spec(), X, y, ln)
    alpha, mll = engine.mll(y)
    assert abs(mll - o["mll"]) <= RTOL * abs(o["mll"])
    assert _rel(alpha, o["alpha"]) < RTOL


def test_gpe_mirror_end_to_end(engine):
    """GPE mirror: dtarget vs finite differences of target (test/kernels.jl:148-164), interpolation
    (test/gp.jl:32-38), optimize! increases the target (test/optim.jl)."""
    import gpb200
    X, _, _ = make_data(200, 2, 4)
    y = np.sin(X.sum(axis=1))
    gp = gpb200.GPE(X.T, y, gpb200.MeanConst(0.1), gpb200.SEIso(0.0, 0.0) + gpb200.fix(gpb200.RQIso(0.3, -1.0, 0.2), "lα"), -2.0,
                    engine=engine)
    gp.update_target_and_dtarget()
    p0 = gp.get_params()
    assert p0.size == 1 + 1 + 2 + 2 and gp.dtarget.size == p0.size
    fd = np.zeros_like(p0)
    for i in range(p0.size):
        for s in (+1, -1):
            p = p0.copy(); p[i] += s * 1e-5
            gp.set_params(p); gp.update_target()
            fd[i] += s * gp.target
        fd[i] /= 2e-5
    gp.set_params(p0); gp.update_target_and_dtarget()
    assert np.allclose(gp.dtarget, fd, rtol=1e-4, atol=1e-4)
    # LOO predictions (test/test_crossvalidation.jl: analytic LOO == refit without point i).  Checked on the initial,
    # well-conditioned hyper-parameters (cond(K_y) ~ 1e4): after optimize() on noiseless data cond(K_y) ~ 1e12 and no two
    # inverses agree to 1e-8.  diag(K_y^-1) is verified by a residual (K_y z_i = e_i  =>  [K^-1]_ii = z_i[i]) rather than
    # against a second explicit inverse.
    mu_loo, s2_loo = gp.predict_LOO()
    Ky = orc.gram(gp.kernel.spec(), X, gp.logNoise)
    r = y - gp.mean.mean(X)
    idx = np.array([0, 17, 63, 128, 199])
    Z = np.linalg.solve(Ky, np.eye(200)[:, idx])
    assert np.max(np.abs(Ky @ Z - np.eye(200)[:, idx])) < 1e-10
    assert np.allclose(1.0 / s2_loo[idx], Z[idx, np.arange(idx.size)], rtol=1e-9)
    Kinv = np.linalg.inv(Ky)
    assert np.allclose(s2_loo, 1.0 / np.diag(Kinv), rtol=1e-8)
    assert np.allclose(mu_loo, y - (Kinv @ r) / np.diag(Kinv), rtol=1e-7, atol=1e-9)
    keep = np.arange(200) != 17
    f17 = orc.fit(gp.kernel.spec(), X[keep], y[keep], gp.logNoise, gp.mean.spec())
    m17, v17 = orc.predict_f(gp.kernel.spec(), X[keep], f17, X[17:18], gp.mean.spec())
    assert abs(mu_loo[17] - m17[0]) < 1e-7 and abs(s2_loo[17] - (v17[0] + gp.noise_variance())) < 1e-7
    assert np.isfinite(gp.logp_LOO())
    t0 = gp.target
    gp.optimize(maxiter=15)
    assert gp.target > t0
    mu, s2 = gp.predict_f(X.T)
    assert np.max(np.abs(mu - y)) < 0.1
    _, cov = gp.predict_f(X.T[:, :9], full_cov=True)
    assert np.allclose(np.diag(cov), s2[:9], atol=1e-8)
    with pytest.raises(ValueError):
        gp.predict_f(np.zeros((3, 5)))
    my, sy = gp.predict_y(X.T[:, :5])
    assert np.allclose(sy, s2[:5] + gp.noise_variance())
    # rand(gp, X, n) (test/gp.jl: posterior samples): right shape, sample mean -> predictive mean
    gp.set_params(p0); gp.update_target()            # back to the well-conditioned initial hyper-parameters
    Xq = X.T[:, :6] + 0.05
    draws = gp.rand(Xq, 4000, rng=np.random.default_rng(0))
    mq, cq = gp.predict_f(Xq, full_cov=True)
    assert draws.shape == (6, 4000)
    assert np.max(np.abs(draws.mean(axis=1) - mq)) < 5 * np.sqrt(np.max(np.diag(cq)) / 4000) + 1e-6


def test_engine_stream_profile_and_options(engine):
    """set_stream (caller-owned CUDA stream), per-launch GEMM profiling counters, option validation, FP64 peak probe."""
    import torch
    import gpb200
    X, y, _ = make_data(900, 3, 77)
    k = gpb200.SEIso(0.2, 0.1)
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    o = orc.fit(k.spec(), X, y, -0.5)
    s = torch.cuda.Stream()
    engine.set_stream(s.cuda_stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    engine.set_option("profile", 1)
    e0.record(s)
    engine.factorize(theta, -0.5)
    alpha, mll = engine.mll(y)
    engine.grad_prepare()
    e1.record(s)
    torch.cuda.synchronize()
    assert e0.elapsed_time(e1) > 0.0
    assert abs(mll - o["mll"]) <= RTOL * abs(o["mll"])
    t = engine.timings()
    assert t["gemm_launches"] > 0 and t["gemm_ms"] > 0 and t["gemm_flops"] > 2.0 * 900 ** 3 / 3
    engine.set_option("profile", 0)
    engine.set_stream(0)
    for lookahead in (0, 1):                                   # both schedules give the same factor bit for bit
        engine.set_option("lookahead", lookahead)
        engine.factorize(theta, -0.5)
        a2, m2 = engine.mll(y)
        assert m2 == mll and np.array_equal(a2, alpha)
    with pytest.raises(ValueError):
        engine.set_option("nb", 300)
    for key, value in (("no_such_option", 1), ("leaf", 0), ("shard_la", 0), ("trsv_fused", 2)):
        with pytest.raises(ValueError):
            engine.set_option(key, value)
    pk = engine.fp64_peak()
    assert 5.0 < pk["dmma_tflops"] < 80.0 and 5.0 < pk["dfma_tflops"] < 80.0
    assert engine.launch_count() > 0


def test_predict_chunking_and_explicit_alpha(engine, monkeypatch):
    """Many test points are streamed through the cross-Gram workspace in chunks; alpha may be passed explicitly."""
    import gpb200
    X, y, _ = make_data(700, 3, 13)
    Xs = np.random.default_rng(14).standard_normal((1000, 3))
    k = gpb200.Mat52Iso(0.1, 0.2)
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    engine.factorize(theta, -0.7)
    alpha, _ = engine.mll(y)
    o = orc.fit(k.spec(), X, y, -0.7)
    mo, vo = orc.predict_f(k.spec(), X, o, Xs)
    monkeypatch.setenv("GPB200_PREDICT_CHUNK", "256")              # 4 chunks of 256 rows
    mu, var, _ = engine.predict(Xs, alpha=o["alpha"])
    assert _rel(mu, mo) < RTOL
    assert np.max(np.abs(var - vo)) <= RTOL * np.max(np.abs(vo)) + 1e-13
    monkeypatch.delenv("GPB200_PREDICT_CHUNK")
    mu1, var1, _ = engine.predict(Xs)                              # single chunk, resident alpha
    assert np.allclose(mu1, mu, rtol=0, atol=1e-12 * np.max(np.abs(mu))) and np.allclose(var1, var, rtol=0, atol=1e-12)


@pytest.mark.parametrize("d,N,ll,ls", [(1, 300, 0.2, 0.1), (2, 515, -0.5, 0.3), (5, 700, 0.4, -0.2), (8, 1300, 0.3, 0.3),
                                       (8, 640, -2.5, 0.0), (3, 500, 0.0, 9.0), (4, 500, 0.5, -9.0)])
def test_seiso_tma_kernels_match_generic_and_oracle(engine, d, N, ll, ls):
    """gram_fast.cu (TMA-staged tiles, table-based exp2) against the generic kernel-program kernels (libm exp) and the
    oracle: Gram entries to 4 ulp of the largest entry, incl. the deep-underflow region (ll = -2.5: exp(-r/2l^2) down to
    1e-300), extreme signal variances, padding tiles and per-point noise; gradient trace to 1e-12."""
    import gpb200
    X, y, _ = make_data(N, d, 31 + d)
    if ll < -2:
        X *= 4.0                                           # push exp arguments below -700
    k = gpb200.SEIso(ll, ls)
    noise = -0.3 + 0.1 * np.cos(np.arange(N))              # VectorParam noise (src/GPE.jl:177-186)
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    res = {}
    for fast in (1, 0):
        engine.set_option("gram_fast", fast)
        engine.factorize(theta, noise)
        K = engine.gram()
        alpha, mll = engine.mll(y)
        engine.grad_prepare()
        g, trA = engine.grad_kernel()
        res[fast] = (K, mll, g, trA)
    engine.set_option("gram_fast", 1)
    Ko = orc.cov(k.spec(), X) + np.diag(np.exp(2 * noise))
    scale = np.max(np.abs(Ko))
    assert np.max(np.abs(res[1][0] - Ko)) <= 1e-15 * scale * 4
    assert np.max(np.abs(res[1][0] - res[0][0])) <= 1e-15 * scale * 4
    # relative accuracy of the small entries too (not only in the max norm): compare where the oracle is > 1e-280
    big = Ko > 1e-280 * np.exp(2 * ls)
    rel = np.abs(res[1][0][big] - Ko[big]) / Ko[big]
    assert np.max(rel) <= 1e-12, np.max(rel)               # |x| * (rounding of r) amplification in the exponent, |x| <= 645
    # mll / gradients inherit cond(K_y): the extreme-variance cases (cond ~ 1e9) only check the Gram entries above
    if abs(ls) < 5:
        assert abs(res[1][1] - res[0][1]) <= 1e-12 * abs(res[0][1])
        assert np.allclose(res[1][2], res[0][2], rtol=1e-10, atol=1e-12 * np.max(np.abs(res[0][2])))
        assert abs(res[1][3] - res[0][3]) <= 1e-10 * abs(res[0][3])
    else:
        assert abs(res[1][1] - res[0][1]) <= 1e-7 * abs(res[0][1])


@pytest.mark.parametrize("M,n", [(37, 5), (300, 130)])
def test_rand_on_device_matches_oracle(engine, M, n):
    """rand(gp, X, n) (src/GP.jl:120-146) on the device: with the SAME standard-normal draws the samples equal
    mu* + chol(Sigma* + nugget I) Z of the oracle's predictMVN (full covariance)."""
    import gpb200
    X, y, _ = make_data(900, 3, 5)
    Xs = np.random.default_rng(8).standard_normal((M, 3)) * 1.5
    k = gpb200.Mat52Iso(0.2, 0.1) + gpb200.SEIso(0.5, -0.5)
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    engine.factorize(theta, -1.0)
    engine.mll(y)
    o = orc.fit(k.spec(), X, y, -1.0)
    mo, co = orc.predict_f(k.spec(), X, o, Xs, full_cov=True)
    z = np.random.default_rng(9).standard_normal((n, M))
    mu, draws = engine.rand(Xs, z, nugget=1e-6)
    L = np.linalg.cholesky(co + 1e-6 * np.eye(M))
    want = mo[None, :] + z @ L.T
    assert _rel(mu, mo) < RTOL
    assert np.max(np.abs(draws - want)) <= 1e-8 * np.max(np.abs(want))
    with pytest.raises(ValueError):
        engine.rand(Xs, z[:, :-1])


def test_crossvalidation_on_device_matches_oracle(engine):
    """src/crossvalidation.jl on the resident inverse: predict_LOO / logp_LOO / dlogpdθ_LOO and predict_CVfold / logp_CVfold /
    dlogpdθ_CVfold (device: K^-1 dK_j K^-1 as two DMMA GEMMs + sub-block gathers; host: the reference's O(N) / per-fold assembly)
    against the oracle's literal restatement (itself pinned to refits and finite differences on the CPU)."""
    import gpb200
    X, y, _ = make_data(420, 2, 17)
    k = gpb200.Mat52Iso(0.3, 0.1) + gpb200.fix(gpb200.SEIso(-0.2, 0.3), "lσ")
    ln = -0.7
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), k, ln, engine=engine)
    gp.update_target_and_dtarget()
    f = orc.fit(k.spec(), X, y, ln)
    mu, s2 = gp.predict_LOO()
    mo, so = orc.predict_loo(f, y)
    assert _rel(mu, mo) < 1e-9 and _rel(s2, so) < 1e-9
    assert abs(gp.logp_LOO() - orc.logp_loo(f, y)) <= 1e-9 * abs(orc.logp_loo(f, y))
    g = gp.dlogp_LOO(noise=True, kern=True)
    go = orc.dlogp_loo(k.spec(), X, y, f, ln)
    assert g.shape == go.shape == (1 + 3,) and np.allclose(g, go, rtol=1e-7, atol=1e-9), (g, go)
    rng = np.random.default_rng(3)
    perm = rng.permutation(420)
    folds = [np.sort(perm[:100]), np.sort(perm[100:250]), np.arange(420)[np.isin(np.arange(420), perm[250:])]]
    mus, Sigs = gp.predict_CVfold(folds)
    muo, Sigo = orc.predict_cvfold(f, y, folds)
    for a, b, c, dd in zip(mus, muo, Sigs, Sigo):
        assert _rel(a, b) < 1e-8 and _rel(c, dd) < 1e-8
    assert abs(gp.logp_CVfold(folds) - orc.logp_cvfold(f, y, folds)) <= 1e-8 * abs(orc.logp_cvfold(f, y, folds))
    gf = gp.dlogp_CVfold(folds, noise=True, kern=True)
    gfo = orc.dlogp_cvfold(k.spec(), X, y, f, ln, folds)
    assert np.allclose(gf, gfo, rtol=1e-6, atol=1e-8), (gf, gfo)
    # the trace-based mll gradient still works after the inverse was mirrored for CV
    gp.update_dmll()
    o = orc.mll_and_dmll(k.spec(), X, y, ln)
    assert np.allclose(gp.dmll, o["dmll"], rtol=1e-8, atol=1e-10)


def test_elastic_append_matches_batch_fit():
    """ElasticGPE append! (src/GPEelastic.jl:13-22; test/elastic.jl:17-29: incremental == batch Cholesky / alpha / mll): the
    device extends its factor in place inside the reserved capacity; beyond it the host mirror refits with more room."""
    import gpb200
    X, y, Xs = make_data(1000, 2, 23, m=40)
    k = gpb200.Mat32Iso(0.3, 0.1) + gpb200.SEIso(0.6, -0.3)
    gp = gpb200.ElasticGPE(X[:300].T, y[:300], gpb200.MeanConst(0.1), k, -0.8, capacity=700, stepsize=200)
    n = 300
    for step in (1, 50, 200, 100, 260):                      # within a tile, across tiles, up to the capacity, beyond it (refit)
        l0 = gp._eng.launch_count()
        gp.append(X[n:n + step].T, y[n:n + step])
        n += step
        assert gp.nobs == n and gp.alpha.size == n
        o = orc.fit(k.spec(), X[:n], y[:n], -0.8, ("MeanConst", 0.1))
        assert abs(gp.mll - o["mll"]) <= 1e-10 * abs(o["mll"]), (step, gp.mll, o["mll"])
        assert _rel(gp.alpha, o["alpha"]) < 1e-10
        mu, s2 = gp.predict_f(Xs.T)
        mo, vo = orc.predict_f(k.spec(), X[:n], o, Xs, ("MeanConst", 0.1))
        assert _rel(mu, mo) < 1e-10 and np.max(np.abs(s2 - vo)) <= 1e-10 * np.max(np.abs(vo)) + 1e-13
    # the gradient path works on the extended factor
    gp.update_dmll()
    og = orc.mll_and_dmll(k.spec(), X[:n], y[:n], -0.8, ("MeanConst", 0.1))
    assert np.allclose(gp.dmll, og["dmll"], rtol=1e-8, atol=1e-10)
    with pytest.raises(ValueError):
        gp.append(np.zeros((3, 2)), [0.0, 1.0])


def test_diagonal_tile_kernel_matches_oracle(engine):
    """potrf_base.cu: the blocked 128 x 128 leaf (16-column panels) against the oracle: factor, inverted tiles (through
    solve / K^-1), log-determinant."""
    import gpb200
    X, y, _ = make_data(1000, 3, 41)
    k = gpb200.Mat52Iso(0.0, 0.2) + gpb200.SEIso(0.4, -0.1)
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    o = orc.fit(k.spec(), X, y, -1.2)
    engine.factorize(theta, -1.2)
    U = engine.factor_upper()
    alpha, mll = engine.mll(y)
    engine.grad_prepare()
    ld, Kinv = engine.logdet(), engine.inverse()
    Ky = orc.gram(k.spec(), X, -1.2)
    assert np.max(np.abs(U.T @ U - Ky)) <= 1e-12 * np.max(np.abs(Ky))
    assert abs(mll - o["mll"]) <= RTOL * abs(o["mll"]) and _rel(alpha, o["alpha"]) < RTOL
    assert abs(ld - np.linalg.slogdet(Ky)[1]) <= 1e-11 * abs(ld)
    assert np.max(np.abs(Kinv @ Ky - np.eye(1000))) <= 1e-9


def test_triangular_solve_variants_agree(engine):
    """alpha = K_y^-1 r (src/GPE.jl:208) through the two schedules of the blocked solves: one launch per block step and
    the single-launch kernels (diagonal tile in registers, neighbour tile in shared memory) -- same arithmetic order, so
    the results agree bit for bit; both match the oracle."""
    import gpb200
    X, y, _ = make_data(3000, 3, 51)
    k = gpb200.SEIso(0.2, 0.1) + gpb200.Mat12Iso(0.5, -0.4)
    theta, _ = _setup(engine, k, X, nb=0, gemm=0)
    engine.factorize(theta, -0.9)
    o = orc.fit(k.spec(), X, y, -0.9)
    res = {}
    for v in (0, 1):
        engine.set_option("trsv_fused", v)
        alpha, mll = engine.mll(y)
        res[v] = (alpha, mll, engine.solve(np.cos(X[:, 1])))
        assert _rel(alpha, o["alpha"]) < RTOL and abs(mll - o["mll"]) <= RTOL * abs(o["mll"])
    assert np.array_equal(res[0][0].view(np.uint64), res[1][0].view(np.uint64))
    assert np.array_equal(res[0][2].view(np.uint64), res[1][2].view(np.uint64)) and res[0][1] == res[1][1]
