"""CPU: the numpy model of the sparse engine's non-GEMM kernels (tests/sparse_model.py) against independent statements:

* the FSA layout's block-diagonal products equal dense products with scipy.linalg.block_diag, and its Gram / gradient
  tile lists cover every block's lower triangle / whole block exactly once;
* the cross-validation row kernels, composed chunk by chunk with the schedule's GEMMs, reproduce the schedule model
  tests/fitc_cv_model.py (itself tested against the dense inverse of Sigma);
* the exact kernel programs are exact on dyadic inputs (float64 == long double) and agree with the oracle;
* the float64 model lies within the stated bounds of the long-double one;
* no output changes when every element a kernel must not read is NaN."""
import numpy as np
import pytest
import scipy.linalg as sl

import sparse_model as sm
import vec_model as vm
from fitc_cv_model import SparseCV
from oracle import gp_oracle as orc

T = sm.T
SIZES = [0, 1, 127, 128, 129, 300, 1100, 2048]
NAN = np.nan


def _packed(rng, lay):
    return rng.standard_normal(lay.packed)


def test_layout_tables():
    lay = sm.Layout(SIZES)
    assert lay.bsize == [0, 128, 128, 128, 256, 384, 1152, 2048]
    assert lay.Np == sum(lay.bsize) and lay.packed == sum(B * B for B in lay.bsize)
    for b, (n, B) in enumerate(zip(SIZES, lay.bsize)):
        P = lay.bstart[b]
        assert np.all(lay.rblk[P:P + B] == b) and lay.boff[b] == sum(c * c for c in lay.bsize[:b])
        assert np.all(lay.mask[P:P + n] == 1) and np.all(lay.mask[P + n:P + B] == 0)
    assert np.array_equal(np.sort(lay.pos), np.flatnonzero(lay.mask))
    perm = np.random.default_rng(0).permutation(lay.N)
    lp = sm.Layout(SIZES, perm)
    assert np.array_equal(lp.pos[perm], lay.pos[np.arange(lay.N)])


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_bdmv_equals_block_diag_products(mode):
    rng = np.random.default_rng(mode)
    lay = sm.Layout(SIZES)
    pk = _packed(rng, lay)
    v = rng.standard_normal(lay.Np)
    got = sm.bdmv(mode, pk, lay, v)
    if mode == 2:
        want = np.sum(lay.dense(pk, "lower") ** 2, axis=1)
    else:
        want = lay.dense(pk, "lower" if mode == 0 else "upper") @ v
    assert np.allclose(got, want, rtol=1e-13, atol=1e-12)
    blocks = [sl.block_diag(np.tril(lay.block(pk, b))) for b in range(len(SIZES)) if lay.bsize[b]]
    assert lay.dense(pk, "lower").shape == (lay.Np, lay.Np) and len(blocks) == 7


def test_gram_items_cover_each_lower_triangle_once_and_gtiles_each_block():
    lay = sm.Layout(SIZES)
    low = np.zeros(lay.packed, int)
    full = np.zeros(lay.packed, int)
    for items, cnt in ((lay.gram_items(), low), (lay.gtiles(), full)):
        for off, ld, ri, rj, diag in items:
            b = lay.rblk[ri]
            assert lay.rblk[rj] == b and ld == lay.bsize[b]
            for i in range(T):
                w = np.arange(T) <= i if diag else np.ones(T, bool)
                cnt[off + i * ld:off + i * ld + T][w] += 1
    for b, B in enumerate(lay.bsize):
        if B:
            assert np.array_equal(lay.block(low, b), np.tril(np.ones((B, B), int)))
            assert np.array_equal(lay.block(full, b), np.ones((B, B), int))
    assert all(d == (ri == rj) for _, _, ri, rj, d in lay.gram_items())


@pytest.mark.parametrize("spec,d", [(("Sum", ("LinIso", [0.0]), ("Const", [0.0])), 3), (("LinArd", [0.0] * 5), 5),
                                    (("Poly", [0.0, 0.0], 2), 3),
                                    (("Prod", ("Poly", [0.0, 0.0], 2), ("Sum", ("LinArd", [0.0] * 3), ("Const", [0.0]))), 3)])
def test_exact_programs_are_exact_and_match_the_oracle(spec, d):
    rng = np.random.default_rng(d)
    X1, X2 = vm.dyadic(rng, (40, d)), vm.dyadic(rng, (30, d))
    K, g = sm.kprog(spec, X1, X2, grad=True)
    Kl, gl = sm.kprog(spec, X1, X2, np.longdouble, grad=True)
    assert np.array_equal(K, Kl.astype(np.float64)) and all(np.array_equal(a, b.astype(np.float64)) for a, b in zip(g, gl))
    Ko, go = orc.cov_and_grads(spec, X1, X2, True)
    assert np.array_equal(K, Ko) and len(g) == len(go) and all(np.array_equal(a, b) for a, b in zip(g, go))


def _sparse_cv(mode="FITC"):
    rng = np.random.default_rng(3)
    N, M, d = 300, 20, 2
    X, Xu = rng.uniform(-2, 2, (N, d)), rng.uniform(-2, 2, (M, d))
    spec = ("SEIso", [0.1, 0.2])
    return SparseCV(spec, X, Xu, -1.0, mode, chunk=128), rng


def _diag_grad(spec, Xc, param):
    return np.array([orc.cov_and_grads(spec, Xc[i:i + 1], Xc[i:i + 1], True)[1][param][0, 0] for i in range(Xc.shape[0])])


@pytest.mark.parametrize("mode", ["FITC", "DTC"])
@pytest.mark.parametrize("param", [0, 1, -1])
def test_row_kernels_composed_reproduce_the_schedule_model(mode, param):
    m, rng = _sparse_cv(mode)
    N, Mu = m.X.shape[0], m.Xu.shape[0]
    alpha = rng.standard_normal(N)
    want_zja, want_dg = m.cv_param(param, alpha)
    noise = param < 0
    kind = 2 if noise else (0 if mode == "FITC" else 1)
    Dp = np.zeros((Mu, Mu)) if noise else m.gKuu[param] @ m.A
    R, H = np.zeros((Mu, Mu)), np.zeros((Mu, Mu))
    kta, gta, uD = np.zeros(Mu), np.zeros(Mu), np.zeros(Mu)
    dl_all = np.empty(N)
    chunks = list(m._chunks(0 if noise else param))
    for r0, K, dK, Xc in chunks:                                    # pass 1
        nc = K.shape[0]
        sl_ = slice(r0, r0 + nc)
        lam, a = m.lam[sl_], alpha[sl_]
        G = None if noise else dK - 0.5 * K @ Dp.T
        dk = np.zeros(nc) if kind else _diag_grad(m.spec, Xc, param)
        rp = -(-nc // T) * T
        dl, da = sm.delta(kind, dk, G, K @ m.A, Mu, nc, rp, np.concatenate([a, np.full(rp - nc, NAN)]),
                          np.full(rp, NAN), np.full(rp, NAN))
        assert np.all(da[nc:] == 0) and np.all(np.isnan(dl[nc:]))
        dl_all[sl_] = dl[:nc]
        KL = K / lam[:, None]
        kta += K.T @ a
        uD += KL.T @ da[:nc]
        gta += (np.zeros_like(K) if noise else G).T @ a
        R += KL.T @ (np.zeros_like(K) if noise else G)
        H += KL.T @ (KL * dl[:nc, None])
    beta = m.A @ kta
    w = sm.wvec(gta, uD, R @ beta, Mu, np.full(Mu, NAN))
    Q = sm.qs(H, R, Mu, np.full((Mu, Mu), NAN))
    zja, dg = np.empty(N), np.empty(N)
    for r0, K, dK, Xc in chunks:                                    # pass 2
        nc = K.shape[0]
        sl_ = slice(r0, r0 + nc)
        lam = m.lam[sl_]
        Ch = (K @ m.B) / lam[:, None]
        G = None if noise else dK - 0.5 * K @ Dp.T
        zja[sl_], dg[sl_] = sm.rows(G, Ch, K, Ch @ Q, nc, Mu, lam, dl_all[sl_], alpha[sl_], beta, w)
    for got, want in ((zja, want_zja), (dg, want_dg)):
        assert np.max(np.abs(got - want)) <= 1e-10 * np.max(np.abs(want)), np.max(np.abs(got - want))
    # the fold block of the same parameter, on duplicated and unsorted indices
    V = np.array([17, 3, 250, 3, 128, 127, 299])
    nv = V.size
    xg, lamg, delg = sm.gather(V, m.X, m.X.shape[1], m.lam, dl_all, nv, np.full((nv + 1, 3), NAN), np.full(nv + 1, NAN),
                               np.full(nv + 1, NAN))
    assert np.all(np.isnan(xg[:, 2])) and np.isnan(lamg[nv]) and np.isnan(delg[nv])
    xg, lamg, delg = xg[:nv, :2], lamg[:nv], delg[:nv]
    K, gK = orc.cov_and_grads(m.spec, xg, m.Xu, True)
    Ch = (K @ m.B) / lamg[:, None]
    G = None if noise else gK[param] - 0.5 * K @ Dp.T
    E = sm.eblock(0.5 * Ch @ Q, G, K, nv, Mu, lamg, delg)
    out1 = sm.diag(E @ Ch.T + Ch @ E.T, nv, 1, lamg, delg)
    out0 = sm.diag(-Ch @ (K / lamg[:, None]).T, nv, 0, lamg, None)
    for which, got in ((1, out1), (0, out0)):
        want = m.cv_block(which, V)
        assert np.max(np.abs(got - want)) <= 1e-10 * np.max(np.abs(want)), (which, np.max(np.abs(got - want)))
    # the inverse diagonal
    q = np.concatenate([np.sum(K * (K @ m.B), axis=1) for _, K in m._chunks()])
    assert np.allclose(sm.invdiag(m.lam, q, N, np.full(N, NAN)), m.inverse_diag(), rtol=1e-12, atol=0)


def test_float64_model_within_bounds_of_long_double():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")
    rng = np.random.default_rng(9)
    lay = sm.Layout([1, 129, 300])
    pk, v = _packed(rng, lay), rng.standard_normal(lay.Np)
    for mode in (0, 1, 2):
        err = np.abs(sm.bdmv(mode, pk, lay, v) - sm.bdmv(mode, pk, lay, v, np.longdouble))
        assert np.all(err <= sm.bdmv_bound(mode, pk, lay, v)), mode
    A, vv = rng.standard_normal((T, 300)), rng.standard_normal(300)
    for sq in (0, 1):
        err = np.abs(sm.rowdot(A, vv, 257, sq) - sm.rowdot(A, vv, 257, sq, np.longdouble))
        assert np.all(err <= sm.rowdot_bound(A, vv, 257, sq)), sq
    G, C, dk, a = rng.standard_normal((50, 40)), rng.standard_normal((50, 40)), rng.standard_normal(50), rng.standard_normal(50)
    f = sm.delta(0, dk, G, C, 37, 50, 64, a, np.zeros(64), np.zeros(64))[0][:50]
    ld = sm.delta(0, dk, G, C, 37, 50, 64, a, np.zeros(64), np.zeros(64), np.longdouble)[0][:50]
    assert np.all(np.abs(f - ld) <= sm.delta_bound(dk, G, C, 37, 50))
    spec = ("SEArd", [0.1, -0.2, 0.3, 0.0])
    gfun = lambda X1, X2: orc.cov_and_grads(spec, X1, X2, True)[1]
    xb = rng.standard_normal((lay.Np, 3))
    items = lay.gtiles()
    W = rng.standard_normal(lay.packed)
    f = sm.trace(gfun, xb, items, lay.mask, W, 4)
    ld = sm.trace(gfun, xb, items, lay.mask, W, 4, np.longdouble)
    assert np.all(np.abs(f - ld) <= sm.trace_bound(gfun, xb, items, lay.mask, W, 4))


def test_unread_elements_do_not_change_the_model():
    rng = np.random.default_rng(5)
    lay = sm.Layout([1, 129, 300])
    spec = ("Sum", ("LinIso", [0.0]), ("Const", [0.0]))
    kf = lambda X1, X2: sm.kprog(spec, X1, X2)[0]
    gf = lambda X1, X2: sm.kprog(spec, X1, X2, grad=True)[1]
    xb = vm.dyadic(rng, (lay.Np, 2))
    xn = np.where(lay.mask[:, None] != 0, xb, NAN)                  # padding rows are never evaluated
    dst = vm.dyadic(rng, lay.packed)
    assert np.array_equal(sm.gram(kf, xb, lay.gram_items(), lay.mask, 0.5, dst), sm.gram(kf, xn, lay.gram_items(), lay.mask, 0.5, dst))
    W = vm.dyadic(rng, lay.packed)
    Wn = W.copy()
    for off, ld, ri, rj, _ in lay.gtiles():
        for i in range(T):
            Wn[off + i * ld:off + i * ld + T][(lay.mask[ri + i] == 0) | (lay.mask[rj:rj + T] == 0)] = NAN
    assert np.array_equal(sm.trace(gf, xb, lay.gtiles(), lay.mask, W, 2), sm.trace(gf, xn, lay.gtiles(), lay.mask, Wn, 2))
    xs = vm.dyadic(rng, (lay.Np, 2))
    assert np.array_equal(sm.crossgram(kf, xs, xb, lay.gtiles()[:3], lay.mask, dst),
                          sm.crossgram(kf, xs, xn, lay.gtiles()[:3], lay.mask, dst))
    pk = vm.dyadic(rng, lay.packed)
    v = vm.dyadic(rng, lay.Np)
    for mode, part in ((0, "upper"), (1, "lower"), (2, "upper")):
        pn = pk.copy()
        for b, B in enumerate(lay.bsize):
            blk = lay.block(pn, b)
            blk[np.triu_indices(B, 1) if part == "upper" else np.tril_indices(B, -1)] = NAN
        assert np.array_equal(sm.bdmv(mode, pk, lay, v), sm.bdmv(mode, pn, lay, None if mode == 2 else v))
    A = vm.dyadic(rng, (T, 40))
    An = A.copy()
    An[:, 33:] = NAN
    vn = np.concatenate([A[0, :33], np.full(7, NAN)])
    for sq in (0, 1):
        assert np.array_equal(sm.rowdot(A, A[0], 33, sq), sm.rowdot(An, vn, 33, sq))
    G, C = vm.dyadic(rng, (9, 40)), vm.dyadic(rng, (9, 40))
    Gn, Cn = G.copy(), C.copy()
    Gn[:, 37:], Cn[:, 37:], Gn[7:], Cn[7:] = NAN, NAN, NAN, NAN
    a = vm.dyadic(rng, 9)
    an = a.copy()
    an[7:] = NAN
    dk = vm.dyadic(rng, 9)
    z = np.zeros(9)
    for want, got in zip(sm.delta(0, dk, G, C, 37, 7, 9, a, z, z), sm.delta(0, dk, Gn, Cn, 37, 7, 9, an, z, z)):
        assert np.array_equal(want, got)
    lam = np.array([0.5, 2.0, 4.0, 1.0, 0.25, 8.0, 2.0, NAN, NAN])
    K = vm.dyadic(rng, (9, 40))
    bw = vm.dyadic(rng, 40)
    bwn = np.concatenate([bw[:37], np.full(3, NAN)])
    Kn = np.where(Gn == Gn, K, NAN)
    r1 = sm.rows(G, C, K, K, 7, 37, lam, dk, a, bw, bw)
    r2 = sm.rows(Gn, Cn, Kn, Kn, 7, 37, lam, dk, an, bwn, bwn)
    assert all(np.array_equal(x, y) for x, y in zip(r1, r2))
    E = vm.dyadic(rng, (9, 40))
    assert np.array_equal(sm.eblock(E, G, K, 7, 37, lam, dk), sm.eblock(E, Gn, Kn, 7, 37, lam, dk))
    assert np.array_equal(sm.eblock(E, None, K, 7, 37, lam, dk), sm.eblock(E, None, Kn, 7, 37, lam, dk))
    Rm = vm.dyadic(rng, (6, 6))
    Rn = Rm.copy()
    Rn[5:, :], Rn[:, 5:] = NAN, NAN
    assert np.array_equal(sm.qs(Rm, Rm, 5, Rm)[:5, :5], sm.qs(Rn, Rn, 5, Rm)[:5, :5])
    S = vm.dyadic(rng, (6, 6))
    Sn = S.copy()
    Sn[np.triu_indices(6, 1)] = NAN
    Sn[5:, :] = NAN
    assert np.array_equal(sm.symmetrize(S, 5)[:5, :5], sm.symmetrize(Sn, 5)[:5, :5])
