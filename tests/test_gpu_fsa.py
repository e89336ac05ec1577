"""GPU: the Full Scale Approximation (mode 3 of the sparse engine, src/sparse/full_scale_approximation.jl) through the C ABI
against the blockwise CPU oracle (tests/fsa_oracle.py).  Tolerances follow test_gpu_fitc.py: max(1e-10, C cond(K_uu) eps),
with cond measured and printed next to the observed errors."""
import math

import numpy as np
import pytest

from oracle import gp_oracle as orc
from fsa_oracle import fsa_dmll_kern, fsa_fit, fsa_predict_closed, fsa_predict_full, nearest_blocks

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _cond_kuu(spec, Xu):
    w = np.linalg.eigvalsh(orc.cov(spec, Xu) + 1e-10 * np.eye(Xu.shape[0]))
    return float(w[-1] / w[0])


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def _check(gp, o, spec, X, Xu, what, C_s=4.0, C_v=64.0):
    cond = _cond_kuu(spec, Xu)
    tol_s, tol_v = max(1e-10, C_s * cond * EPS), max(1e-10, C_v * cond * EPS)
    e_mll = abs(gp.mll - o["mll"]) / abs(o["mll"])
    e_ld = abs(gp.logdet - o["logdet"]) / abs(o["logdet"])
    e_al = _rel(gp.alpha, o["alpha"])
    e_dn = abs(gp.dmll[0] - o["dmll_noise"]) / abs(o["dmll_noise"])
    print("FSA %s: cond(K_uu+1e-10I)=%.2e  mll %.2e logdet %.2e alpha %.2e dmll_noise %.2e  (bounds %.1e / %.1e)"
          % (what, cond, e_mll, e_ld, e_al, e_dn, tol_s, tol_v))
    assert e_mll <= tol_s and e_ld <= tol_s + 1e-12
    assert e_al <= tol_v
    assert e_dn <= max(1e-9, 16 * tol_v)
    gk = fsa_dmll_kern(spec, X, Xu, o)
    nk = gk.size
    e_gk = _rel(gp.dmll[-nk:], gk)
    print("    kernel gradient %.2e: %s" % (e_gk, np.array2string(gp.dmll[-nk:], precision=6)))
    assert np.allclose(gp.dmll[-nk:], gk, rtol=max(1e-6, 16 * tol_v), atol=1e-7)     # as test_gpu_fitc.py


def _check_predict(gp, o, spec, X, Xu, Xs, bpred, mspec, what, full=True):
    """predict_f with and without full_cov, and predict_y, against the closed form the GPU evaluates (fsa_predict_closed) and
    against the literal predictMVN (:413-447).  The two oracles differ by the effect of Sigma_QR's second 1e-10 nugget
    (:227), which the closed form's S = K_uu + K_uf Lambda^-1 K_fu does not carry: ~1e-10 / lambda_min(K_uu) relative."""
    mo, So = fsa_predict_closed(spec, X, Xu, o, Xs, bpred, mspec)
    ml, Sl = fsa_predict_full(spec, X, Xu, o, Xs, bpred, mspec)
    cond = _cond_kuu(spec, Xu)
    tol = max(1e-9, 64.0 * cond * EPS)
    mu, s2 = gp.predict_f(Xs.T, bpred)
    scale = float(np.max(np.abs(So)))
    e_mu, e_var = _rel(mu, mo), float(np.max(np.abs(s2 - np.maximum(np.diag(So), 0.0)))) / scale
    e_lit = float(np.max(np.abs(s2 - np.maximum(np.diag(Sl), 0.0)))) / scale
    print("FSA predict %s: mu %.2e var %.2e (bound %.1e); var vs the literal predictMVN %.2e" % (what, e_mu, e_var, tol, e_lit))
    assert e_mu <= tol and e_var <= tol
    assert _rel(mu, ml) <= 1e-6 and e_lit <= 1e-6
    my, sy = gp.predict_y(Xs.T, bpred)
    assert np.array_equal(my, mu) and np.allclose(sy, s2 + gp.noise_variance(), rtol=1e-15, atol=0)
    if full:
        mu2, S = gp.predict_f(Xs.T, bpred, full_cov=True)
        e_S = float(np.max(np.abs(S - So))) / float(np.max(np.abs(So)))
        print("    full_cov %.2e" % e_S)
        assert _rel(mu2, mo) <= tol and e_S <= tol


def _fd_gradient(gp, h):
    """central differences of the GPU mll over [logNoise; mean; kernel], the order of update_dmll"""
    import gpb200 as g

    def mll_at(ln, mp, kp):
        gp.logNoise = ln
        if mp is not None:
            gp.mean.set_params(mp)
        gp.kernel.set_params(kp)
        gp.update_mll()
        return gp.mll

    ln0, mp0, kp0 = gp.logNoise, list(gp.mean.get_params()), list(gp.kernel.get_params())
    params = [ln0] + mp0 + kp0
    nm = len(mp0)
    out = []
    for i in range(len(params)):
        vals = []
        for sgn in (1, -1):
            q = list(params)
            q[i] += sgn * h
            vals.append(mll_at(q[0], q[1:1 + nm] if nm else None, q[1 + nm:]))
        out.append((vals[0] - vals[1]) / (2 * h))
    mll_at(ln0, mp0 if nm else None, kp0)
    return np.array(out)


def _mixed_blocks(N, sizes, rng):
    perm = rng.permutation(N)
    out, p = [], 0
    for s in sizes:
        out.append(np.sort(perm[p:p + s])); p += s
    while p < N:
        s = min(400, N - p)
        out.append(perm[p:p + s]); p += s
    return out


def test_fsa_reference_config():
    """test/test_sparse.jl:15-36, 158-160: N = 1000, d = 1, 12 quantile inducing points, blocks by nearest inducing point"""
    import gpb200 as g
    rng = np.random.default_rng(1)
    x = rng.beta(7, 7, 1000) * 10
    y = np.abs(x - 5) * np.cos(2 * x) + rng.normal(0, 10.0, 1000)
    X = x[:, None]
    Xu = np.quantile(x, [0.2, 0.25, 0.3, 0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65, 0.7, 0.98])[:, None]
    blocks = nearest_blocks(X, Xu)
    k = g.SEIso(math.log(0.3), math.log(5.0))
    m = g.MeanConst(float(np.mean(y)))
    gp = g.FSA(X.T, Xu.T, blocks, y, m, k, math.log(10.0))
    gp.update_dmll()
    o = fsa_fit(k.spec(), X, Xu, blocks, y, math.log(10.0), ("MeanConst", float(np.mean(y))))
    _check(gp, o, k.spec(), X, Xu, "reference config")
    assert abs(gp.dmll[1] - o["dmll_mean"][0]) <= 1e-7 * abs(o["dmll_mean"][0]) + 1e-9
    xtest = rng.beta(7, 7, 30) * 10                                           # test_sparse.jl:33, 84-87
    _check_predict(gp, o, k.spec(), X, Xu, xtest[:, None], nearest_blocks(xtest[:, None], Xu), ("MeanConst", float(np.mean(y))),
                   "reference config")
    full = orc.fit(k.spec(), X, y, math.log(10.0), ("MeanConst", float(np.mean(y))))
    assert abs(gp.mll - full["mll"]) <= 10.0                                   # test_sparse.jl:158-160 (FSA vs exact)
    # [noise; mean; kernel] against central differences of the GPU mll (test_sparse.jl:137-145: atol 1e-3)
    fd = _fd_gradient(gp, h=1e-4)
    print("    central differences:", fd, "analytical:", gp.dmll)
    assert np.allclose(gp.dmll, fd, rtol=0, atol=1e-3)


def test_fsa_mixed_block_sizes():
    import gpb200 as g
    rng = np.random.default_rng(7)
    sizes = [0, 1, 127, 128, 129, 300, 1100, 2048]
    N, M, d = 6000, 150, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    blocks = _mixed_blocks(N, sizes, rng)
    k = g.Mat32Iso(-0.3, 0.0) + g.RQIso(-0.5, -0.5, 0.3)
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanConst(0.1), k, -1.0)
    gp.update_dmll()
    o = fsa_fit(k.spec(), X, Xu, blocks, y, -1.0, ("MeanConst", 0.1))
    _check(gp, o, k.spec(), X, Xu, "mixed blocks N=%d M=%d" % (N, M))
    # test blocks: 300 points paired with the 2048-point block (3 test tiles), a few with every other block, some unpaired,
    # and test blocks past the last training block (no Lambda_xf term, like zip)
    Xs = rng.standard_normal((520, d))
    bpred = [np.arange(300 + j * j, 300 + j * j + j) for j in range(7)] + [np.arange(0, 300)] + [np.arange(350, 360)]
    bpred += [np.array([], dtype=np.int64)] * (len(blocks) - len(bpred)) + [np.arange(360, 390)]
    _check_predict(gp, o, k.spec(), X, Xu, Xs, bpred, ("MeanConst", 0.1), "mixed blocks")


def test_fsa_one_block_is_the_exact_gp():
    """one block holding every point: Sigma = K + (sigma^2 + 1e-10) I, the exact GP (GPE with the 1e-10 nugget)"""
    import gpb200 as g
    rng = np.random.default_rng(3)
    N, d = 1500, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-1.5, 1.5, 5)
    Xu = np.array([[a, b] for a in grid for b in grid])
    k = g.SEIso(-0.2, 0.1)
    gp = g.FSA(X.T, Xu.T, [rng.permutation(N)], y, g.MeanConst(0.1), k, -1.0)
    gp.update_dmll()
    e = orc.mll_and_dmll(k.spec(), X, y, -1.0, ("MeanConst", 0.1), extra_nugget=1e-10)
    print("FSA one block: mll %.2e alpha %.2e dmll %.2e" % (abs(gp.mll - e["mll"]) / abs(e["mll"]), _rel(gp.alpha, e["alpha"]),
                                                           _rel(gp.dmll, e["dmll"])))
    assert abs(gp.mll - e["mll"]) <= 1e-9 * abs(e["mll"])
    assert _rel(gp.alpha, e["alpha"]) <= 1e-9
    assert np.allclose(gp.dmll, e["dmll"], rtol=1e-8, atol=1e-8), (gp.dmll, e["dmll"])
    # GPE has no 1e-10 nugget: the two mll differ by about 1e-10 tr(K_y^-1) / 2
    Xs = rng.standard_normal((64, d))
    mu, S = gp.predict_f(Xs.T, [np.arange(64)], full_cov=True)
    mo, So = orc.predict_f(k.spec(), X, e, Xs, ("MeanConst", 0.1), full_cov=True)
    print("    predict vs exact GP: mu %.2e cov %.2e" % (_rel(mu, mo), _rel(S, So)))
    assert _rel(mu, mo) <= 1e-9 and _rel(S, So) <= 1e-9
    ref = g.GPE(X.T, y, g.MeanConst(0.1), k, -1.0)
    ref.update_mll()
    tr_kinv = float(e["alpha"] @ e["alpha"] - e["trA"])
    assert abs(gp.mll - ref.mll) <= 1e-10 * tr_kinv + 1e-9 * abs(ref.mll)


def test_fsa_singleton_blocks_are_fitc():
    import gpb200 as g
    rng = np.random.default_rng(5)
    N, d = 3000, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-2.0, 2.0, 6)
    Xu = np.array([[a, b] for a in grid for b in grid])
    k = g.SEIso(-0.5, 0.0)
    gp = g.FSA(X.T, Xu.T, [np.array([i]) for i in range(N)], y, g.MeanZero(), k, -1.0)
    gp.update_dmll()
    f = g.FITC(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    f.update_dmll()
    o = fsa_fit(k.spec(), X, Xu, [np.array([i]) for i in range(N)], y, -1.0)
    _check(gp, o, k.spec(), X, Xu, "singleton blocks")
    # FITC's Lambda has no 1e-10 block nugget: the mll differ by ~1e-10 tr(Sigma^-1) / 2 <= 1e-10 N / (2 sigma^2)
    assert abs(gp.mll - f.mll) <= 1e-10 * N * math.exp(2.0) + 1e-9 * abs(f.mll)
    assert np.allclose(gp.dmll, f.dmll, rtol=1e-6, atol=1e-6), (gp.dmll, f.dmll)


def test_fsa_chunked():
    """N = 70 000, M = 64, blocks of ~500: several staging chunks"""
    import gpb200 as g
    rng = np.random.default_rng(11)
    N, M, d = 70000, 64, 2
    X = rng.uniform(-3, 3, (N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    order = np.argsort(X[:, 0] + 0.3 * X[:, 1])
    blocks = [order[i:i + 500] for i in range(0, N, 500)]
    k = g.SEIso(-0.5, 0.0)
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), k, -1.0)
    gp.update_dmll()
    o = fsa_fit(k.spec(), X, Xu, blocks, y, -1.0)
    _check(gp, o, k.spec(), X, Xu, "chunked N=%d" % N)
    # 600 test points paired with the training blocks, then the same points among 40 000 unpaired ones: more padded test rows
    # than one staging chunk, so the test rows are streamed too
    Xs = rng.uniform(-3, 3, (600, d))
    ob = np.argsort(Xs[:, 0] + 0.3 * Xs[:, 1])
    bpred = [ob[j * 4:(j + 1) * 4] for j in range(len(blocks))][:150]
    _check_predict(gp, o, k.spec(), X, Xu, Xs, bpred, ("MeanZero",), "chunked", full=False)
    Xbig = np.concatenate([Xs, rng.uniform(-3, 3, (40000, d))])
    mu_b, s2_b = gp.predict_f(Xbig.T, bpred)
    mu_s, s2_s = gp.predict_f(Xs.T, bpred)
    assert _rel(mu_b[:600], mu_s) <= 1e-12 and _rel(s2_b[:600], s2_s) <= 1e-12
    mo, So = fsa_predict_closed(k.spec(), X, Xu, o, Xbig[-200:], [])
    assert _rel(mu_b[-200:], mo) <= 1e-9 and float(np.max(np.abs(s2_b[-200:] - np.maximum(np.diag(So), 0)))) <= 1e-9 * float(np.max(So))


def test_fsa_finite_differences_seard():
    """SEArd d = 3, N = 6000: every parameter against central differences of the GPU mll.  The inducing points lie on a
    4 x 4 x 4 grid: with a well-conditioned K_uu (cond ~ 1e3) the second 1e-10 nugget of Sigma_QR (:227), which the analytical
    gradient does not see, moves the mll by far less than the difference tolerance (with random inducing points,
    cond ~ 1e8, it does not: test_sparse.jl allows 1e-3)."""
    import gpb200 as g
    rng = np.random.default_rng(19)
    N, d = 6000, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-1.8, 1.8, 4)
    Xu = np.array([[a, b, c] for a in grid for b in grid for c in grid])
    order = np.argsort(X[:, 0])
    blocks = [order[i:i + 700] for i in range(0, N, 700)]
    k = g.SEArd([-0.2, 0.1, 0.3], 0.2)
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanConst(0.1), k, -1.0)
    gp.update_dmll()
    fd = _fd_gradient(gp, h=1e-4)
    print("FSA SEArd: analytical", gp.dmll, "central differences", fd)
    assert np.allclose(gp.dmll, fd, rtol=1e-6, atol=1e-6)


def test_fsa_launch_count_does_not_depend_on_the_number_of_blocks():
    """equal N, M and largest block, 16 blocks vs 241 blocks: the same number of launches for factorize + mll + gradient"""
    import gpb200 as g
    rng = np.random.default_rng(13)
    N, M, d = 32768, 64, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1))
    Xu = X[:M]
    perm = rng.permutation(N)
    counts = []
    for blocks in ([perm[i:i + 2048] for i in range(0, N, 2048)],
                   [perm[:2048]] + [perm[i:i + 128] for i in range(2048, N, 128)]):
        gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.SEIso(-0.5, 0.0), -1.0)
        c0 = gp._eng.launch_count()
        gp.update_mll()
        gp.update_dmll()
        counts.append(gp._eng.launch_count() - c0)
    print("launches: %d blocks -> %d, %d blocks -> %d" % (16, counts[0], 241, counts[1]))
    assert counts[0] == counts[1]


def test_fsa_error_paths_leave_the_handle_usable():
    import gpb200 as g
    from gpb200.capi import FitcEngine
    rng = np.random.default_rng(17)
    N, M, d = 2100, 20, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1))
    Xu = X[:M]
    k = g.SEIso(-0.5, 0.0)
    ops, dims, theta, _ = g.flatten(k, d)
    eng = FitcEngine(0)
    eng.set_mode(3)
    eng.set_data(np.ascontiguousarray(X), np.ascontiguousarray(Xu))
    eng.set_kernel(ops, dims, theta.size)
    with pytest.raises(ValueError, match="set_blocks"):
        eng.factorize(theta, -1.0)                                           # GPB200_ESTATE: no blocks yet
    with pytest.raises(ValueError, match="2048"):
        eng.set_blocks(np.array([0, N]), np.arange(N))                       # one block of 2100 > 2048 points
    with pytest.raises(ValueError, match="partition"):
        eng.set_blocks(np.array([0, 300, N]), np.concatenate([np.arange(300), np.arange(299, N - 1)]))
    blocks = nearest_blocks(X, Xu)
    bp = np.concatenate([[0], np.cumsum([b.size for b in blocks])])
    eng.set_blocks(bp, np.concatenate(blocks))
    eng.factorize(theta, -1.0)
    alpha, mll, ld = eng.mll(y)
    with pytest.raises(ValueError, match="test blocks"):
        eng.predict(np.ascontiguousarray(X[:5]))
    with pytest.raises(ValueError, match="test blocks"):
        eng.predict_cov(np.ascontiguousarray(X[:5]))
    o = fsa_fit(k.spec(), X, Xu, blocks, y, -1.0)
    assert abs(mll - o["mll"]) <= 1e-9 * abs(o["mll"])
    assert _rel(alpha, o["alpha"]) <= 1e-7
    eng.close()
