"""CPU: the numpy model of the triangular solves, the GPA kernels and the reductions (tests/vec_model.py) means what the
engine needs -- the blocked recurrences are triangular solves with the dense L whose diagonal tiles are inv(Dinv), the scan
gives S = W'Z = W' M_s W (the identity at the top of csrc/gpa.cu), the float64 model stays within the derived bounds of
the long-double one, and nothing changes when every element the model says is unread holds a NaN."""
import numpy as np
import pytest
import scipy.linalg as sl

import vec_model as vm

T = vm.T


def _need_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")


def _factor(N, seed=0, nug=1e-3):
    """lower Cholesky factor of an SE Gram matrix, padded to Npad with identity rows (as the engine pads), and the float64
    inverted diagonal tiles"""
    rng = np.random.default_rng(seed)
    x = np.sort(rng.uniform(0, 8, N))
    K = np.exp(-0.5 * (x[:, None] - x[None, :]) ** 2) + nug * np.eye(N)
    Npad = -(-N // T) * T
    L = np.eye(Npad)
    L[:N, :N] = np.linalg.cholesky(K)
    Dinv = np.zeros((Npad, T))
    for b in range(Npad // T):
        s = slice(b * T, (b + 1) * T)
        Dinv[s] = sl.solve_triangular(L[s, s], np.eye(T), lower=True)
    return L, Dinv, rng


def _poison_solve(L):
    F = np.where(vm.trsv_read_mask(L.shape[0], L.shape[0]), L, np.nan)
    return F


@pytest.mark.parametrize("N", [300, 384, 700])
def test_blocked_solves_are_triangular_solves_with_inv_dinv_tiles(N):
    _need_longdouble()
    L, Dinv, rng = _factor(N, seed=N)
    Npad = L.shape[0]
    Ld = L.copy()                       # the dense L the recurrences solve with: diagonal tiles inv(Dinv)
    for b in range(Npad // T):
        s = slice(b * T, (b + 1) * T)
        Ld[s, s] = np.tril(np.linalg.inv(Dinv[s]))
    F = _poison_solve(L)
    r = np.zeros(Npad)
    r[:N] = rng.standard_normal(N)
    y, _ = vm.trsv_fwd(F, Dinv, r, np.longdouble)
    ref = sl.solve_triangular(Ld, r, lower=True)
    assert np.max(np.abs(np.float64(y) - ref)) <= 1e-10 * np.max(np.abs(ref))
    a, _ = vm.trsv_bwd(F, vm.transpose_tiles(Dinv), r, np.longdouble)
    ref = sl.solve_triangular(Ld.T, r, lower=False)
    assert np.max(np.abs(np.float64(a) - ref)) <= 1e-10 * np.max(np.abs(ref))
    # and both together solve K_y
    y64, _ = vm.trsv_fwd(F, Dinv, r)
    a64, _ = vm.trsv_bwd(F, vm.transpose_tiles(Dinv), y64)
    K = L @ L.T
    assert np.max(np.abs(K @ a64 - r)) <= 1e-8 * np.max(np.abs(r))


def test_exact_solve_construction_returns_the_planted_solution():
    rng = np.random.default_rng(5)
    nb = 6
    Npad = nb * T
    Ld, W = vm.exact_diag_tiles(rng, nb)
    for ld in (Npad, Npad + 256, T):
        flat = vm.dyadic(rng, (Npad - 1) * ld + Npad)
        F = np.lib.stride_tricks.as_strided(flat, shape=(Npad, Npad), strides=(8 * ld, 8), writeable=False)
        y = rng.integers(-4, 5, Npad).astype(np.float64)
        r = vm.lower_product(F, Ld, y)
        got, acc = vm.trsv_fwd(F, W, r)
        assert np.array_equal(got, y)
        for b in range(nb):                 # what the per-step schedule leaves in r: L_bb y_b
            s = slice(b * T, (b + 1) * T)
            assert np.array_equal(acc[s], Ld[s] @ y[s])
        z = vm.lower_t_product(F, Ld, y)
        got, _ = vm.trsv_bwd(F, vm.transpose_tiles(W), z)
        assert np.array_equal(got, y)


def test_scan_gives_w_transpose_ms_w():
    """S = W'Z (lower part) = W' M_s W with M_s[i, j] = u[max(i, j)] v[min(i, j)]"""
    _need_longdouble()
    L, Dinv, rng = _factor(300, seed=3, nug=1e-2)
    Npad = L.shape[0]
    W = sl.solve_triangular(L, np.eye(Npad), lower=True)
    tb = np.arange(Npad) // T
    G = np.where(tb[None, :] > tb[:, None], W.T, np.nan)          # W' in G's strict-upper tiles only
    DinvT = vm.transpose_tiles(np.vstack([W[b * T:(b + 1) * T, b * T:(b + 1) * T] for b in range(Npad // T)]))
    u, v = rng.standard_normal(Npad), rng.standard_normal(Npad)
    Zf, ZdT = vm.gpa_scan(G, DinvT, u, v, np.longdouble)
    fw, _ = vm.scan_masks(Npad, Npad)
    assert np.all(Zf[~fw] == 0)
    for b in range(Npad):
        assert np.all(ZdT[b, :b % T] == 0)
    Z = vm.scan_lower_Z(np.float64(Zf), np.float64(ZdT))
    i = np.arange(Npad)
    Ms = u[np.maximum(i[:, None], i[None, :])] * v[np.minimum(i[:, None], i[None, :])]
    S = np.tril(W.T @ Z)
    ref = np.tril(W.T @ Ms @ W)
    assert np.max(np.abs(S - ref)) <= 1e-9 * np.max(np.abs(ref))
    # Z itself: the definition at the top of csrc/gpa.cu, column by column
    for b in (0, 1, 127, 128, 200, Npad - 1):
        for c in (b, min(b + 1, Npad - 1), Npad - 1):
            want = u[c] * np.sum(v[b:c + 1] * W[b:c + 1, b]) + v[c] * np.sum(u[c + 1:] * W[c + 1:, b])
            assert abs(Z[c, b] - want) <= 1e-12 * (1 + abs(want))


def test_models_ignore_every_unread_element():
    rng = np.random.default_rng(7)
    Npad = 3 * T
    F = rng.standard_normal((Npad, Npad + 64))
    D = rng.standard_normal((Npad, T))
    r = rng.standard_normal(Npad)
    Fp = np.where(vm.trsv_read_mask(Npad, Npad + 64), F, np.nan)
    for fn in (vm.trsv_fwd, vm.trsv_bwd):
        a, b = fn(F, D, r), fn(Fp, D, r)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    Fp = np.where(vm.trmv_read_mask(Npad, Npad + 64), F, np.nan)
    for fn in (vm.trmv, vm.trmv_t):
        assert np.array_equal(fn(F, r), fn(Fp, r))
    fw, dr = vm.scan_masks(Npad, Npad + 64)
    u, v = rng.standard_normal(Npad), rng.standard_normal(Npad)
    a = vm.gpa_scan(F, D, u, v)
    b = vm.gpa_scan(np.where(fw, F, np.nan), np.where(dr, D, np.nan), u, v)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    x, y = rng.standard_normal(2000), rng.standard_normal(2000)
    xp, yp = x.copy(), y.copy()
    xp[1500:] = np.nan
    yp[1500:] = np.nan
    assert vm.dot(x, y, 1500) == vm.dot(xp, yp, 1500) and vm.vsum(x, 1500) == vm.vsum(xp, 1500)
    K = rng.standard_normal((5, 300))
    Kp = K.copy()
    Kp[:, 257:] = np.nan
    assert np.array_equal(vm.rowdot(K, x, 4, 257), vm.rowdot(Kp, xp[:257].copy(), 4, 257))
    assert np.array_equal(vm.rowvar(K, y, 4, 257), vm.rowvar(Kp, y, 4, 257))
    assert np.array_equal(vm.rowdot2(K, 2 * K, 4, 257), vm.rowdot2(Kp, 2 * Kp, 4, 257))


def test_float64_model_within_the_derived_bounds():
    """the bounds hold for one concrete float64 evaluation order (numpy's), and they are not vacuous: the float64 error
    reaches a visible fraction of them"""
    _need_longdouble()
    L, Dinv, rng = _factor(640, seed=11, nug=1e-4)
    Npad = L.shape[0]
    F = _poison_solve(L)
    r = rng.standard_normal(Npad)
    ratios = []
    y, _ = vm.trsv_fwd(F, Dinv, r)
    ref, bnd = vm.trsv_fwd_local(F, Dinv, r, y)
    ratios.append(np.max(np.abs(y - ref) / bnd))
    a, _ = vm.trsv_bwd(F, vm.transpose_tiles(Dinv), r)
    ref, bnd = vm.trsv_bwd_local(F, vm.transpose_tiles(Dinv), r, a)
    ratios.append(np.max(np.abs(a - ref) / bnd))
    ratios.append(np.max(np.abs(vm.trmv(L, r) - vm.trmv(L, r, np.longdouble)) / vm.trmv_bound(L, r)))
    ratios.append(np.max(np.abs(vm.trmv_t(L, r) - vm.trmv_t(L, r, np.longdouble)) / vm.trmv_t_bound(L, r)))
    G, D = rng.standard_normal((Npad, Npad)), rng.standard_normal((Npad, T))
    u, v = rng.standard_normal(Npad), rng.standard_normal(Npad)
    fw, _ = vm.scan_masks(Npad, Npad)
    (zf, zd), (zfl, zdl), (bf, bd) = vm.gpa_scan(G, D, u, v), vm.gpa_scan(G, D, u, v, np.longdouble), vm.gpa_scan_bound(G, D, u, v)
    ratios.append(max(np.max(np.abs(zf - zfl)[fw] / bf[fw]), np.max(np.abs(zd - zdl) / np.where(bd > 0, bd, np.inf))))
    x, w = rng.standard_normal(100000), rng.standard_normal(100000)
    ratios.append(abs(vm.dot(x, w, x.size) - vm.dot(x, w, x.size, np.longdouble)) / vm.dot_bound(x, w, x.size))
    ratios.append(abs(vm.vsum(x, x.size) - vm.vsum(x, x.size, np.longdouble)) / vm.vsum_bound(x, x.size))
    K = rng.standard_normal((4, 5000))
    ratios.append(np.max(np.abs(vm.rowdot(K, x, 4, 5000) - vm.rowdot(K, x, 4, 5000, np.longdouble)) / vm.rowdot_bound(K, x, 4, 5000)))
    ratios.append(np.max(np.abs(vm.rowvar(K, w, 4, 5000) - vm.rowvar(K, w, 4, 5000, np.longdouble)) / vm.rowvar_bound(K, w, 4, 5000)))
    ratios.append(np.max(np.abs(vm.rowdot2(K, K[::-1], 4, 5000) - vm.rowdot2(K, K[::-1], 4, 5000, np.longdouble))
                         / vm.rowdot2_bound(K, K[::-1], 4, 5000)))
    assert max(ratios) <= 1.0, ratios
    assert max(ratios) > 1e-6, ratios


def test_exact_operands_make_every_reduction_exact():
    """dyadic operands j/256 with n = 10^6: every partial sum is a multiple of 2^-16 below 2^20, so float64 equals long
    double whatever the order"""
    _need_longdouble()
    rng = np.random.default_rng(9)
    n = 10 ** 6
    a, b = vm.dyadic(rng, n), vm.dyadic(rng, n)
    assert vm.dot(a, b, n) == vm.dot(a, b, n, np.longdouble)
    assert vm.dot(a[::-1].copy(), b[::-1].copy(), n) == vm.dot(a, b, n)
    assert vm.vsum(a, n) == vm.vsum(a, n, np.longdouble)
