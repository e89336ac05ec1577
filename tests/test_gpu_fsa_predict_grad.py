"""GPU: FSA's predictive gradients (gpb200_fitc_predict_fsa_grad, FSA.predict_f_grad(x, blockindpred)) against the CPU
restatement fsa_xgrad_oracle.fsa_predict_f_grad, the exact GP and FITC in their limits, central differences of the device
predictions, and the contraction kernel fsa_crossgram_dx on caller buffers.  Error bound: max(1e-8, 64 cond(K_uu) eps) of
the largest entry, the bound of test_gpu_fitc_predict_grad.py; cond(K_uu) and the largest cond(Lambda_b) are printed."""
import math
import zlib

import numpy as np
import pytest

from conftest import kernel_zoo, make_data
from fsa_oracle import fsa_fit, fsa_predict_closed, nearest_blocks
from oracle import gp_oracle as orc
import xgrad_oracle as xo
from fsa_xgrad_oracle import fsa_predict_f_grad

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _cond_kuu(spec, Xu):
    w = np.linalg.eigvalsh(orc.cov(spec, Xu) + 1e-10 * np.eye(Xu.shape[0]))
    return float(w[-1] / w[0])


def _cond_lam(o):
    return max((float(np.linalg.cond(U)) ** 2 for U in o["Ulam"] if U.size), default=1.0)


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def _parity(gp, o, spec, X, Xu, Xs, bpred, mspec, what):
    """device (raw and through FSA.predict_f_grad) against the oracle; mu / var bitwise those of predict_fsa; repeated
    calls and the call without var bitwise equal"""
    from gpb200.sparse import test_block_of
    cond = _cond_kuu(spec, Xu)
    tol = max(1e-8, 64.0 * cond * EPS)
    mo, vo, dmo, dvo = fsa_predict_f_grad(spec, X, Xu, o, Xs, bpred, mspec)
    xs = np.ascontiguousarray(Xs)
    bo = test_block_of(bpred, Xs.shape[0])
    e = gp._eng
    mu, var, dmu, dvar = e.predict_fsa_grad(xs, bo)
    mean = gp.mean.mean(xs)
    errs = (_rel(mu + mean, mo), _rel(var, vo), _rel(dmu + gp.mean.grad_x(xs), dmo), _rel(dvar, dvo))
    print("FSA predict_f_grad %s: cond(K_uu)=%.2e max cond(Lambda_b)=%.2e  mu %.2e var %.2e dmu %.2e dvar %.2e (bound %.1e)"
          % (what, cond, _cond_lam(o), *errs, tol))
    assert max(errs) <= tol, errs
    m0, v0 = e.predict_fsa(xs, bo)
    assert np.array_equal(mu, m0) and np.array_equal(var, v0)
    m1, v1, dm1, dv1 = e.predict_fsa_grad(xs, bo)
    assert all(np.array_equal(a, b) for a, b in ((mu, m1), (var, v1), (dmu, dm1), (dvar, dv1)))
    m2, v2, dm2, dv2 = e.predict_fsa_grad(xs, bo, want_var=False)
    assert v2 is None and dv2 is None and np.array_equal(m2, mu) and np.array_equal(dm2, dmu)
    mu_h, s2_h, dmu_h, ds2_h = gp.predict_f_grad(Xs.T, bpred)
    assert dmu_h.shape == (Xs.shape[1], Xs.shape[0]) and np.array_equal(s2_h, np.maximum(var, 0.0))
    return mu, var, dmu, dvar


def test_fsa_predict_grad_reference_config():
    """test/test_sparse.jl's configuration: d = 1, 12 quantile inducing points, blocks by nearest inducing point"""
    import gpb200 as g
    rng = np.random.default_rng(1)
    x = rng.beta(7, 7, 1000) * 10
    y = np.abs(x - 5) * np.cos(2 * x) + rng.normal(0, 10.0, 1000)
    X = x[:, None]
    Xu = np.quantile(x, [0.2, 0.25, 0.3, 0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65, 0.7, 0.98])[:, None]
    blocks = nearest_blocks(X, Xu)
    k = g.SEIso(math.log(0.3), math.log(5.0))
    mspec = ("MeanConst", float(np.mean(y)))
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanConst(mspec[1]), k, math.log(10.0))
    o = fsa_fit(k.spec(), X, Xu, blocks, y, math.log(10.0), mspec)
    xtest = np.concatenate([rng.beta(7, 7, 30) * 10, [x[blocks[4][0]]]])      # the last: a training input of its block
    bpred = nearest_blocks(xtest[:30, None], Xu)
    bpred[4] = np.append(bpred[4], 30)
    _parity(gp, o, k.spec(), X, Xu, xtest[:, None], bpred, mspec, "reference config")


def test_fsa_predict_grad_mixed_block_sizes():
    """test_fsa_mixed_block_sizes' blocks: 300 test points on the 2048-point block (three test tiles), a few on every
    other block, unpaired points, test blocks past the last training block and a test point on a training input"""
    import gpb200 as g
    from test_gpu_fsa import _mixed_blocks
    rng = np.random.default_rng(7)
    sizes = [0, 1, 127, 128, 129, 300, 1100, 2048]
    N, M, d = 6000, 150, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    blocks = _mixed_blocks(N, sizes, rng)
    k = g.Mat32Iso(-0.3, 0.0) + g.RQIso(-0.5, -0.5, 0.3)
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanConst(0.1), k, -1.0)
    o = fsa_fit(k.spec(), X, Xu, blocks, y, -1.0, ("MeanConst", 0.1))
    Xs = rng.standard_normal((520, d))
    Xs[337] = X[blocks[6][17]]                                  # paired with block 6 below
    bpred = [np.arange(300 + j * j, 300 + j * j + j) for j in range(7)] + [np.arange(0, 300)] + [np.arange(350, 360)]
    bpred += [np.array([], dtype=np.int64)] * (len(blocks) - len(bpred)) + [np.arange(360, 390)]
    assert 337 in bpred[6]
    _parity(gp, o, k.spec(), X, Xu, Xs, bpred, ("MeanConst", 0.1), "mixed blocks")


def test_fsa_predict_grad_seard_d3():
    import gpb200 as g
    rng = np.random.default_rng(19)
    N, d = 4000, 3
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-1.8, 1.8, 4)
    Xu = np.array([[a, b, c] for a in grid for b in grid for c in grid])
    order = np.argsort(X[:, 0])
    blocks = [order[i:i + 700] for i in range(0, N, 700)]
    k = g.SEArd([-0.2, 0.1, 0.3], 0.2)
    mspec = ("MeanLin", [0.2, -0.1, 0.3])
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanLin([0.2, -0.1, 0.3]), k, -1.0)
    o = fsa_fit(k.spec(), X, Xu, blocks, y, -1.0, mspec)
    Xs = rng.standard_normal((200, d))
    bpred = [np.arange(j * 25, (j + 1) * 25) for j in range(len(blocks))]
    _parity(gp, o, k.spec(), X, Xu, Xs, bpred, mspec, "SEArd d=3")


def test_fsa_predict_grad_one_block_is_the_exact_gp():
    """one block holding every point: the exact GP's gradients with the 1e-10 nugget"""
    import gpb200 as g
    rng = np.random.default_rng(3)
    N, d = 1500, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-1.5, 1.5, 5)
    Xu = np.array([[a, b] for a in grid for b in grid])
    k = g.SEIso(-0.2, 0.1)
    gp = g.FSA(X.T, Xu.T, [rng.permutation(N)], y, g.MeanConst(0.1), k, -1.0)
    e = orc.fit(k.spec(), X, y, -1.0, ("MeanConst", 0.1), 1e-10)
    Xs = rng.standard_normal((64, d))
    mu, s2, dmu, ds2 = gp.predict_f_grad(Xs.T, [np.arange(64)])
    mo, vo, dmo, dvo = xo.predict_f_grad(k.spec(), X, e, Xs, ("MeanConst", 0.1))
    errs = (_rel(mu, mo), _rel(dmu.T, dmo), _rel(ds2.T, dvo))
    print("FSA one block vs exact GP: mu %.2e dmu %.2e dvar %.2e" % errs)
    assert max(errs) <= 1e-9, errs


def test_fsa_predict_grad_singleton_blocks_are_fitc():
    import gpb200 as g
    rng = np.random.default_rng(5)
    N, d = 3000, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    grid = np.linspace(-2.0, 2.0, 6)
    Xu = np.array([[a, b] for a in grid for b in grid])
    k = g.SEIso(-0.5, 0.0)
    gp = g.FSA(X.T, Xu.T, [np.array([i]) for i in range(N)], y, g.MeanZero(), k, -1.0)
    f = g.FITC(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    Xs = rng.standard_normal((100, d))
    a = gp.predict_f_grad(Xs.T, [])
    b = f.predict_f_grad(Xs.T)
    for u, v in zip(a, b):
        np.testing.assert_allclose(u, v, rtol=1e-6, atol=1e-6 * max(np.max(np.abs(v)), 1e-3))


def test_fsa_predict_grad_chunked():
    """N = 70 000, M = 64, blocks of ~500: 600 paired points among 40 000 unpaired ones stream over several test chunks"""
    import gpb200 as g
    rng = np.random.default_rng(11)
    N, M, d = 70000, 64, 2
    X = rng.uniform(-3, 3, (N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    order = np.argsort(X[:, 0] + 0.3 * X[:, 1])
    blocks = [order[i:i + 500] for i in range(0, N, 500)]
    k = g.SEIso(-0.5, 0.0)
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), k, -1.0)
    o = fsa_fit(k.spec(), X, Xu, blocks, y, -1.0)
    Xs = rng.uniform(-3, 3, (600, d))
    ob = np.argsort(Xs[:, 0] + 0.3 * Xs[:, 1])
    bpred = [ob[j * 4:(j + 1) * 4] for j in range(len(blocks))][:150]
    small = _parity(gp, o, k.spec(), X, Xu, Xs, bpred, ("MeanZero",), "chunked")
    Xbig = np.concatenate([Xs, rng.uniform(-3, 3, (40000, d))])
    from gpb200.sparse import test_block_of
    big = gp._eng.predict_fsa_grad(np.ascontiguousarray(Xbig), test_block_of(bpred, Xbig.shape[0]))
    for a, b in zip(big, small):
        assert _rel(a[:600], b) <= 1e-12
    pick = 600 + rng.choice(40000, 150, replace=False)
    mo, vo, dmo, dvo = fsa_predict_f_grad(k.spec(), X, Xu, o, Xbig[pick], [])
    tol = max(1e-8, 64.0 * _cond_kuu(k.spec(), Xu) * EPS)
    errs = (_rel(big[0][pick], mo), _rel(big[1][pick], vo), _rel(big[2][pick], dmo), _rel(big[3][pick], dvo))
    print("FSA chunked, unpaired sample: mu %.2e var %.2e dmu %.2e dvar %.2e (bound %.1e)" % (*errs, tol))
    assert max(errs) <= tol


def test_fsa_predict_grad_large_directional_differences():
    """N = 200 000, M = 1024, blocks of 512: directional central differences of the device predict_f(x, blockindpred)"""
    import gpb200 as g
    rng = np.random.default_rng(23)
    N, M, d = 200000, 1024, 3
    X = rng.uniform(-2, 2, (N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = X[rng.permutation(N)[:M]]
    order = np.argsort(X[:, 0])
    blocks = [order[i:i + 512] for i in range(0, N, 512)]
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.SEIso(-0.3, 0.0), -1.0)
    Xs = rng.uniform(-2, 2, (256, d))
    bpred = [np.array([], dtype=np.int64)] * 100 + [np.arange(0, 128)] + [np.array([], dtype=np.int64)] * 200 + [np.arange(128, 200)]
    mu, s2, dmu, ds2 = gp.predict_f_grad(Xs.T, bpred)
    v = rng.standard_normal((256, d)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    h = 1e-4
    mp, sp = gp.predict_f((Xs + h * v).T, bpred)
    mm, sm = gp.predict_f((Xs - h * v).T, bpred)
    fd_mu, fd_s2 = (mp - mm) / (2 * h), (sp - sm) / (2 * h)
    an_mu, an_s2 = np.sum(dmu.T * v, axis=1), np.sum(ds2.T * v, axis=1)
    e_mu = float(np.max(np.abs(an_mu - fd_mu))) / max(float(np.max(np.abs(an_mu))), 1.0)
    e_s2 = float(np.max(np.abs(an_s2 - fd_s2))) / max(float(np.max(np.abs(an_s2))), 1e-3)
    print("FSA N=200000 directional differences: mu %.2e var %.2e" % (e_mu, e_s2))
    assert e_mu <= 1e-5 and e_s2 <= 1e-5


def test_fsa_predict_grad_leaves_the_handle_unchanged():
    import gpb200 as g
    rng = np.random.default_rng(29)
    N, M, d = 3000, 40, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1))
    Xu = X[:M]
    blocks = nearest_blocks(X, Xu)
    Xs = rng.standard_normal((50, d))
    bpred = nearest_blocks(Xs, Xu)

    def state(gp):
        gp.update_dmll()
        mu, s2 = gp.predict_f(Xs.T, bpred)
        draws = gp.rand(Xs[:10].T, [np.arange(10)], n=3, rng=np.random.default_rng(0))
        return [gp.dmll.copy(), mu, s2, draws]

    k = g.SEIso(-0.5, 0.0) + g.RQIso(-0.3, -0.5, 0.2)
    a = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), k, -1.0)
    b = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), k, -1.0)
    b.predict_f_grad(Xs.T, bpred)
    b._eng.predict_fsa_grad(np.ascontiguousarray(Xs), np.full(50, 2), want_var=False)
    for u, v in zip(state(a), state(b)):
        assert np.array_equal(u, v)


def test_fsa_predict_grad_error_paths():
    import ctypes as C
    import gpb200 as g
    from gpb200.capi import FitcEngine, _as_dp
    rng = np.random.default_rng(31)
    N, M, d = 1200, 20, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1))
    Xu = X[:M]
    Xs = np.ascontiguousarray(rng.standard_normal((30, d)))
    bo = np.zeros(30, dtype=np.int64)
    fitc = g.FITC(X.T, Xu.T, y, g.MeanZero(), g.SEIso(-0.5, 0.0), -1.0)
    with pytest.raises(ValueError, match="FSA mode"):
        fitc._eng.predict_fsa_grad(Xs, bo)                                   # mode 0
    k = g.SEIso(-0.5, 0.0)
    ops, dims, theta, _ = g.flatten(k, d)
    eng = FitcEngine(0)
    eng.set_mode(3)
    eng.set_data(np.ascontiguousarray(X), np.ascontiguousarray(Xu))
    eng.set_kernel(ops, dims, theta.size)
    blocks = nearest_blocks(X, Xu)
    eng.set_blocks(np.concatenate([[0], np.cumsum([b.size for b in blocks])]), np.concatenate(blocks))
    eng.factorize(theta, -1.0)
    with pytest.raises(ValueError, match="mll"):
        eng.predict_fsa_grad(Xs, bo)                                         # GPB200_ESTATE before mll
    eng.mll(y)
    mu, var, dmu, dvar = (np.empty(30), np.empty(30), np.empty((30, d)), np.empty((30, d)))
    rc = eng._lib.gpb200_fitc_predict_fsa_grad(eng._h, 30, _as_dp(Xs), d, bo.ctypes.data_as(C.POINTER(C.c_int64)),
                                               _as_dp(mu), _as_dp(var), _as_dp(dmu), None)
    assert rc == g.capi.EINVAL                                               # var without dvar
    with pytest.raises(ValueError, match="block_of"):
        eng.predict_fsa_grad(Xs, bo[:29])
    a = eng.predict_fsa_grad(Xs, bo)                                         # still usable
    b = eng.predict_fsa(Xs, bo)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---- the contraction kernel on caller buffers ---------------------------------------------------------------------------

def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _dx_case(d, seed):
    """M = 150 inducing points, a padded training layout of three blocks (128, 256 and 128 padded rows, the padding
    poisoned with NaN in x and alpha and masked), 40 real test points at scattered padded rows of a 300-row chunk whose
    other rows are NaN"""
    rng = np.random.default_rng(seed)
    M, Np, R = 150, 512, 300
    Z = rng.standard_normal((M, d))
    xb = rng.standard_normal((Np, d))
    mask = np.ones(Np)
    for lo, hi in ((100, 128), (128 + 200, 384), (384 + 60, 512)):
        mask[lo:hi] = 0.0
    xb[mask == 0] = np.nan
    alpha = rng.standard_normal(Np); alpha[mask == 0] = np.nan
    rows = np.sort(rng.choice(R, 40, replace=False))
    xs = np.full((R, d), np.nan); xs[rows] = rng.standard_normal((40, d))
    xs[rows[3]] = xb[5]                                                      # a test point on a training input of its block
    W = np.full((R, M), np.nan); S1 = np.full((R, M), np.nan); S2 = np.full((R, M), np.nan)
    for A in (W, S1, S2):
        A[rows] = rng.standard_normal((40, M))
    lde = 256
    E = np.full((R, lde), np.nan)
    E[rows] = rng.standard_normal((40, lde))
    blocks = [(0, 128), (128, 256), (384, 128)]
    items = []
    for t, r in enumerate(rows):
        b0, nb = blocks[t % 3] if t % 4 else (0, 0)                          # every fourth point unpaired
        items.append((int(r), int(39 - t), b0, nb))
    return dict(Z=Z, xb=xb, mask=mask, alpha=alpha, xs=xs, W=W, S1=S1, S2=S2, E=E, lde=lde, items=items, M=M)


def _dx_reference(spec, c, d):
    """the contraction with cov_dx's derivatives, summed in np.longdouble"""
    L = np.longdouble
    n = len(c["items"])
    dmu, dvar = np.zeros((n, d)), np.zeros((n, d))
    for row, out, b0, nb in c["items"]:
        x = c["xs"][row:row + 1]
        _, Du = xo.cov_dx(spec, x, c["Z"])
        gm =(Du[0].astype(L) * (1.0 - c["W"][row]).astype(L)[:, None]).sum(0)       # u = 1
        gv = xo.kdiag_dx(spec, x)[0].astype(L) + (Du[0].astype(L) * (2.0 * (c["S1"][row] - c["S2"][row])).astype(L)[:, None]).sum(0)
        if nb:
            idx = np.arange(b0, b0 + nb)
            idx = idx[c["mask"][idx] != 0]
            _, Db = xo.cov_dx(spec, x, c["xb"][idx])
            gm += (Db[0].astype(L) * c["alpha"][idx].astype(L)[:, None]).sum(0)
            gv += (Db[0].astype(L) * c["E"][row, idx - b0].astype(L)[:, None]).sum(0)
        dmu[out], dvar[out] = gm, gv
    return dmu, dvar


def _dx_zoo():
    out = []
    for d in (1, 3, 8):
        out += [(n, d) for n, _ in kernel_zoo(d)]
    return out


@pytest.mark.parametrize("name,d", _dx_zoo(), ids=["%s-d%d" % z for z in _dx_zoo()])
def test_fsa_crossgram_dx_zoo(name, d):
    import gpb200 as g
    kernel = dict(kernel_zoo(d))[name]
    try:
        ops, dims, theta, _ = g.flatten(kernel, d)
    except Exception as exc:                                                 # a zoo entry that needs more dimensions
        pytest.skip("not defined at d = %d: %s" % (d, exc))
    spec = kernel.spec()
    spec = spec[1] if spec[0] == "Fixed" else spec
    c = _dx_case(d, zlib.crc32(("%s%d" % (name, d)).encode()))
    e = g.Engine(0)
    e.set_kernel(ops, dims, theta.size)
    u = np.ones(c["M"])
    dbuf = {k: _dev(c[k]) for k in ("xs", "Z", "xb", "W", "S1", "S2", "mask", "alpha", "E")}
    du = _dev(u)
    n = len(c["items"])

    def run(items, var=True):
        dmu = _dev(np.full((n, d), np.nan)); dvar = _dev(np.full((n, d), np.nan))
        args = [dbuf["xs"].data_ptr(), dbuf["Z"].data_ptr(), dbuf["xb"].data_ptr(), d, c["M"], du.data_ptr(),
                dbuf["W"].data_ptr(), dbuf["S1"].data_ptr(), dbuf["S2"].data_ptr(), c["M"], dbuf["mask"].data_ptr(),
                dbuf["alpha"].data_ptr(), dbuf["E"].data_ptr(), c["lde"], dmu.data_ptr(), dvar.data_ptr() if var else 0]
        n0 = e.launch_count()
        e.fsa_kernels("crossgram_dx", args + [v for it in items for v in it], theta)
        assert e.launch_count() - n0 == (1 if items else 0)
        return _host(dmu), _host(dvar)

    dmu, dvar = run(c["items"])
    rm, rv = _dx_reference(spec, c, d)
    em = float(np.max(np.abs(dmu - rm))) / max(float(np.max(np.abs(rm))), 1e-300)
    ev = float(np.max(np.abs(dvar - rv))) / max(float(np.max(np.abs(rv))), 1e-300)
    print("fsa_crossgram_dx %s d=%d: dmu %.2e dvar %.2e of the largest entry" % (name, d, em, ev))
    assert np.all(np.isfinite(dmu)) and np.all(np.isfinite(dvar))            # no padding row or masked row reached them
    assert em <= 1e-11 and ev <= 1e-11
    # bitwise repeatable; a row's result does not depend on the items sharing the launch; dmu the same without var
    dm2, dv2 = run(c["items"])
    assert np.array_equal(dm2, dmu) and np.array_equal(dv2, dvar)
    half = c["items"][::3]
    dm3, dv3 = run(list(reversed(half)))
    outs = [it[1] for it in half]
    assert np.array_equal(dm3[outs], dmu[outs]) and np.array_equal(dv3[outs], dvar[outs])
    dm4, dv4 = run(c["items"], var=False)
    assert np.array_equal(dm4, dmu) and np.all(np.isnan(dv4))
    e.close()
