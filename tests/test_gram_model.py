"""CPU: the model of the dense Gram-family kernels (tests/gram_model.py) against the oracles, its float64 evaluation
against long double within its bounds in every edge regime, and its tile layouts against dense matrices."""
import zlib

import numpy as np
import pytest

import gram_model as gm
import xgrad_oracle as xo
from conftest import kernel_zoo
from oracle import gp_oracle as orc


def _need_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")


def _spec(kernel):
    spec = kernel.spec()
    return spec[1] if spec[0] == "Fixed" else spec


ZOO = [(n, k, 3) for n, k in kernel_zoo(3)] + [(n + "(d=8)", k, 8) for n, k in kernel_zoo(8) if "Ard" in n]


@pytest.mark.parametrize("name,kernel,d", ZOO, ids=[z[0] for z in ZOO])
def test_model_matches_oracles_across_the_zoo(name, kernel, d):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    A, B = rng.standard_normal((60, d)), rng.standard_normal((60, d))
    B[5] = A[5]
    P = gm.Prog(kernel, d)
    k, _, g, _ = gm.evaluate(P, A, B, grad=True)
    dx, _ = gm.evaluate_dx(P, A, B)
    K, G = orc.cov_and_grads(_spec(kernel), A, B, True)
    _, D = xo.cov_dx(_spec(kernel), A, B)
    i = np.arange(60)
    assert np.max(np.abs(k - K[i, i])) <= 1e-14 * np.max(np.abs(K))
    assert len(G) == P.n_theta
    for p in range(P.n_theta):
        assert np.max(np.abs(g[p] - G[p][i, i])) <= 1e-14 * max(np.max(np.abs(G[p])), 1e-300), (name, p)
    assert np.max(np.abs(dx - D[i, i])) <= 1e-14 * max(np.max(np.abs(D)), 1e-300)


EDGE = gm.edge_table()


@pytest.mark.parametrize("case", range(len(EDGE)), ids=["%s-%s" % (e[0], e[1]) for e in EDGE])
def test_float64_model_within_its_bounds_against_long_double(case):
    _need_longdouble()
    reg, name, kernel, d, A, B = EDGE[case]
    P = gm.Prog(kernel, d)
    with np.errstate(all="ignore"):
        for grad in (False, True):
            k, bk, g, bg = gm.evaluate(P, A, B, np.float64, grad)
            kl, _, gl, _ = gm.evaluate(P, A, B, gm.LD, grad)
            assert np.all(np.isfinite(k)) and np.all(np.abs(k - kl) <= bk), (reg, name, grad)
            if grad:
                assert np.all(np.isfinite(g)) and np.all(np.abs(g - gl) <= bg), (reg, name)
        dx, bdx = gm.evaluate_dx(P, A, B, np.float64)
        dl, _ = gm.evaluate_dx(P, A, B, gm.LD)
    assert np.all(np.isfinite(dx)) and np.all(np.abs(dx - dl) <= bdx), (reg, name)


def _exact():
    import gpb200 as g
    return gm.Prog(g.LinIso(0.0) + g.Const(0.0), 3)


def _dyadic(rng, shape):
    return rng.integers(-64, 65, size=shape) / 16.0


@pytest.mark.parametrize("N", [1, 129, 300])
def test_layouts_compose_to_the_dense_matrices(N):
    rng = np.random.default_rng(N)
    P, d = _exact(), 3
    T = gm.T
    Npad = -(-N // T) * T
    ldx, ld = d + 2, Npad + 4
    x = np.full((Npad, ldx), np.nan)
    x[:N, :d] = _dyadic(rng, (N, d))
    X = x[:N, :d]
    K = gm.kmat(P, X, X)
    kf = lambda a, b: gm.kmat(P, a, b)
    full = np.eye(Npad)
    full[:N, :N] = K + 0.25 * np.eye(N)
    # every ownership split of the lower tiles adds up to the whole lower triangle once
    for own_tiles, nranks, axis in ((0, 1, 0), (1, 3, 0), (1, 3, 1), (2, 2, 1)):
        acc = np.zeros(Npad * ld)
        for rank in range(nranks):
            G = gm.gram_lower(kf, x.ravel(), ldx, d, N, Npad, [0.25], 1, 0.0, np.zeros(Npad * ld), ld, own_tiles, nranks,
                              rank, axis)
            acc += G
        M = acc.reshape(Npad, ld)[:, :Npad]
        lowt = np.kron(np.tril(np.ones((Npad // T, Npad // T))), np.ones((T, T))) > 0
        assert np.array_equal(M[lowt], full[lowt]) and np.all(M[~lowt] == 0)
    # gradient row batches compose to dK/dtheta_j
    gf = lambda a, b: gm.gmat(P, a, b)[0]
    D = np.concatenate([gm.gram_grad_full(gf, x.ravel(), ldx, d, N, Npad, np.zeros(T * ld), ld, r0, T).reshape(T, ld)
                        for r0 in range(0, Npad, T)])
    want = np.zeros((Npad, Npad))
    want[:N, :N] = gm.gmat(P, X, X)[0]
    assert np.array_equal(D[:, :Npad], want)
    # the mirror of the lower tiles gives the full symmetric matrix
    F = gm.mirror_lower_tiles(np.where(lowt, full, np.nan).reshape(-1) if ld == Npad else
                              np.pad(np.where(lowt, full, np.nan), ((0, 0), (0, ld - Npad))).reshape(-1), ld, Npad)
    Fm = F.reshape(Npad, ld)[:, :Npad]
    offdiag = np.kron(1 - np.eye(Npad // T), np.ones((T, T))) > 0
    assert np.array_equal(Fm[offdiag], full[offdiag])
    # trace = sum_{i >= j} w_ij dK_ij, w = A (0.5 A on the diagonal), A = alpha alpha' - Kinv; last entry tr(A)
    alpha = _dyadic(rng, N)
    Kinv = _dyadic(rng, (N, N))
    Kinv = Kinv + Kinv.T
    kb = np.full((Npad, ld), np.nan)
    kb[:N, :N] = Kinv
    A = np.outer(alpha, alpha) - Kinv
    W = np.tril(A, -1) + 0.5 * np.diag(np.diag(A))
    gall = lambda a, b: gm.gmat(P, a, b)
    _, out = gm.trace_out(gm.trace(gall, x.ravel(), ldx, d, N, Npad, alpha, kb.ravel(), ld), P.n_theta)
    Gd = gm.gmat(P, X, X)
    want = [np.sum(W * Gd[p]) for p in range(P.n_theta)] + [np.trace(A)]
    assert np.array_equal(out, want)
    # rectangular trace and the diagonal gradient
    N2 = max(N // 2, 1)
    ldw = N2 + (N2 & 1) + 2
    Wr = np.full((N, ldw), np.nan)
    Wr[:, :N2] = _dyadic(rng, (N, N2))
    _, out = gm.trace_rect(gall, x.ravel(), ldx, N, x.ravel(), ldx, N2, d, Wr.ravel(), ldw, P.n_theta)
    Gr = gm.gmat(P, X, X[:N2])
    assert np.array_equal(out, [np.sum(Wr[:, :N2] * Gr[p]) for p in range(P.n_theta)])
    gv = _dyadic(rng, N)
    kd = gm.kdiag_grad(lambda a, b: np.stack([np.diag(m) for m in gm.gmat(P, a, b)]), x.ravel(), ldx, d, N, gv, P.n_theta)
    assert np.array_equal(kd.reshape(P.n_theta, N), gv[None, :] * np.stack([np.diag(m) for m in Gd]))


def test_nan_in_unread_elements_changes_nothing():
    rng = np.random.default_rng(3)
    P, d, N, T = _exact(), 3, 200, gm.T
    Npad, ldx, ld = 256, 5, 260
    kf, gall = (lambda a, b: gm.kmat(P, a, b)), (lambda a, b: gm.gmat(P, a, b))
    base = np.zeros((Npad, ldx))
    base[:N, :d] = _dyadic(rng, (N, d))
    alpha = np.zeros(Npad)
    alpha[:N] = _dyadic(rng, N)
    Kb = np.zeros((Npad, ld))
    Kb[:N, :N] = np.tril(_dyadic(rng, (N, N)))
    Wb = np.zeros((N, ld))
    Wb[:, :101] = _dyadic(rng, (N, 101))
    runs = []
    for fill in (0.0, np.nan):
        x = base.copy()
        x[N:] = fill
        x[:, d:] = fill
        a = alpha.copy()
        a[N:] = fill
        K = Kb.copy()
        K[:, N + 1:] = fill
        K[np.triu_indices(Npad, 2)] = fill          # read as pairs: only (i, i + 1) of an even row i next to the diagonal
        K[N:] = fill
        W = Wb.copy()
        W[:, 101:] = fill                           # the odd column 101 is read as a pair and discarded
        G = gm.gram_lower(kf, x.ravel(), ldx, d, N, Npad, [0.5], 1, 0.0, np.zeros(Npad * ld), ld)
        C = gm.crossgram(kf, x.ravel(), ldx, N, Npad, x.ravel(), ldx, N, Npad, d, np.zeros(Npad * ld), ld)
        _, tr = gm.trace_out(gm.trace(gall, x.ravel(), ldx, d, N, Npad, a, K.ravel(), ld), P.n_theta)
        _, trr = gm.trace_rect(gall, x.ravel(), ldx, N, x.ravel(), ldx, 101, d, W.ravel(), ld, P.n_theta)
        runs.append((G, C, tr, trr))
    for u, v in zip(*runs):
        assert np.array_equal(u, v)
