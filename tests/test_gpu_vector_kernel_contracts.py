"""GPU: the O(N^2) / O(N) kernels that turn the factor into numbers, tested directly against the model tests/vec_model.py.

* Blocked triangular solves (csrc/vec.cu) through gpb200_trsv_tiles: both schedules (one launch per block step, and the
  single flag-synchronised launch), both directions, nb from 1 to the selection limit 4 x SMs.
* GPA kernels (csrc/gpa.cu) through gpb200_gpa_kernels: f = L v, u = L' g and the prefix / suffix scan that builds Z'.
* Fixed-order reductions (dot, sum, rowdot, rowvar, rowdot2) through gpb200_row_reductions.

Exact cases use dyadic operands j / 256 (|j| <= 256) and small integers: every product and every partial sum is exact in
binary64, so any correct kernel matches the model bit for bit whatever its summation order.  Every element the operation
must not read holds a NaN (F's upper triangle and diagonal tiles for the solves, everything past n or N for the
reductions), and every element it must not write holds a NaN with its own payload that must come back unchanged.
Gaussian cases and real factors from factorize are checked against the long-double model within the derived bounds.

The solves above about 2 x SMs blocks store F with leading dimension 128, so that rows overlap (row j is the run
flat[128 j .. 128 j + Npad)): F is only read, and the model reads the same strided view.

The file sorts after every file that opens a torch.profiler session (torch.profiler records no device activity in a
session started about a minute or more after the process's first one); it opens none itself."""
import numpy as np
import pytest

import vec_model as vm

pytestmark = pytest.mark.gpu

T = vm.T
POISON = np.array([0x7FF8_DEAD_0000_0002], dtype=np.uint64).view(np.float64)[0]   # "never read, never written"


def _bits(a):
    a = np.where(a == 0, 0.0, a)                 # +0 and -0 are the same result of an exact sum
    return np.ascontiguousarray(a).view(np.uint64)


def _raw(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


def _sms():
    return _torch().cuda.get_device_properties(0).multi_processor_count


def _need_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")


def _tail(a, extra):
    """a followed by `extra` POISON elements along axis 0"""
    return np.concatenate([a, np.full((extra,) + a.shape[1:], POISON)])


# ---- triangular solves ------------------------------------------------------------------------------------------------

class _F:
    """F on the host (a view the model reads) and on the device"""

    def __init__(self, rng, nb, layout, fill=None):
        Npad = nb * T
        if layout == "overlap":
            self.ld = T
            self.flat = vm.dyadic(rng, (Npad - 1) * T + Npad)
            self.view = np.lib.stride_tricks.as_strided(self.flat, shape=(Npad, Npad), strides=(8 * T, 8), writeable=False)
        else:
            self.ld = Npad + (256 if layout == "wide" else 0)
            m = vm.trsv_read_mask(Npad, self.ld)
            full = np.full((Npad, self.ld), POISON)
            full[m] = (vm.dyadic(rng, (Npad, self.ld)) if fill is None else fill)[m]
            self.flat = full.ravel()
            self.view = full
        self.dev = _dev(self.flat)


def _trsv(engine, sched, direction, F, D, rhs):
    """one call: returns (out, rhs after, D after, watchdog), checking the launch count and the poisoned tails"""
    Npad = rhs.shape[0]
    dD, dr, do = _dev(_tail(D, T)), _dev(_tail(rhs, T)), _dev(np.full(Npad + T, POISON))
    n0 = engine.launch_count()
    wd = engine.trsv_tiles(sched, direction, [F.dev.data_ptr(), F.ld, dD.data_ptr(), dr.data_ptr(), do.data_ptr(), Npad])
    assert engine.launch_count() - n0 == (1 if sched else Npad // T)
    out, r_after, D_after = _host(do), _host(dr), _host(dD)
    assert wd == 0
    assert np.array_equal(_raw(out[Npad:]), _raw(np.full(T, POISON)))
    assert np.array_equal(_raw(r_after[Npad:]), _raw(np.full(T, POISON)))
    assert np.array_equal(_raw(D_after), _raw(_tail(D, T)))
    return out[:Npad], r_after[:Npad]


def _solve_exact(engine, nb, layout, seed):
    rng = np.random.default_rng(seed)
    Npad = nb * T
    F = _F(rng, nb, layout)
    Ld, W = vm.exact_diag_tiles(rng, nb)
    WT = vm.transpose_tiles(W)
    y = rng.integers(-4, 5, Npad).astype(np.float64)
    cases = ((0, vm.lower_product(F.view, Ld, y), W, vm.trsv_fwd), (1, vm.lower_t_product(F.view, Ld, y), WT, vm.trsv_bwd))
    for direction, rhs, D, model in cases:
        want, acc = model(F.view, D, rhs)
        assert np.array_equal(want, y)                 # the construction: exact operands return the planted solution
        for sched in (0, 1):
            out, r_after = _trsv(engine, sched, direction, F, D, rhs)
            bad = _bits(out) != _bits(want)
            assert not bad.any(), (nb, layout, sched, direction, int(bad.sum()), np.argwhere(bad)[0])
            # the single launch only reads rhs; the per-step schedule leaves r_b - sum L_bi y_i in it
            assert np.array_equal(_bits(r_after), _bits(acc if sched == 0 else rhs)), (nb, layout, sched, direction)
    if layout != "overlap":
        assert np.array_equal(_raw(_host(F.dev)), _raw(F.flat))          # F is only read


@pytest.mark.parametrize("nb", [1, 2, 3, 24])
def test_trsv_exact_full_factor_poisoned(engine, nb):
    _solve_exact(engine, nb, "full", seed=nb)


def test_trsv_exact_ldf_above_npad(engine):
    _solve_exact(engine, 5, "wide", seed=50)


@pytest.mark.parametrize("which", ["24", "SMs-1", "SMs", "SMs+1", "2SMs", "4SMs"])
def test_trsv_exact_overlapping_rows_up_to_the_selection_limit(engine, which):
    s = _sms()
    nb = {"24": 24, "SMs-1": s - 1, "SMs": s, "SMs+1": s + 1, "2SMs": 2 * s, "4SMs": 4 * s}[which]
    _solve_exact(engine, nb, "overlap", seed=nb)


def _real_factor(N, seed):
    import gpb200 as g
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 6, (N, 2))
    eng = g.Engine(0)
    try:
        eng.set_data(X)
        ops, dims, theta, _ = g.flatten(g.SEIso(0.3, 0.0) + g.Mat32Iso(0.8, -0.5), 2)
        eng.set_kernel(ops, dims, theta.size)
        eng.factorize(theta, -3.0)
        L = eng.factor_upper().T
    finally:
        eng.close()
    return L, rng


@pytest.mark.parametrize("N", [1000, 1152, 3000])
def test_trsv_real_factor_within_bound_and_schedules_bitwise(engine, N):
    """L from factorize (identity padding as the engine pads), Dinv = the rounded inverse diagonal tiles; Gaussian
    right-hand side zero in the padding.  Each block is checked against the long-double step from the device's own
    earlier blocks; the two schedules agree bit for bit."""
    _need_longdouble()
    import scipy.linalg as sl
    Lr, rng = _real_factor(N, seed=N)
    Npad = -(-N // T) * T
    L = np.eye(Npad)
    L[:N, :N] = Lr
    D = np.vstack([sl.solve_triangular(L[b * T:(b + 1) * T, b * T:(b + 1) * T], np.eye(T), lower=True)
                   for b in range(Npad // T)])
    DT = vm.transpose_tiles(D)
    F = _F(rng, Npad // T, "full", fill=L)
    r = np.zeros(Npad)
    r[:N] = rng.standard_normal(N)
    for direction, Dd, local in ((0, D, vm.trsv_fwd_local), (1, DT, vm.trsv_bwd_local)):
        outs = [_trsv(engine, sched, direction, F, Dd, r)[0] for sched in (0, 1)]
        assert np.array_equal(_raw(outs[0]), _raw(outs[1])), (N, direction, int(np.sum(outs[0] != outs[1])))
        ref, bnd = local(F.view, Dd, r, outs[1])
        ratio = float(np.max(np.abs(outs[1] - ref) / np.where(bnd > 0, bnd, np.inf)))
        print("RATIO trsv N=%d dir=%d max|err|/bound = %.3e" % (N, direction, ratio))
        assert np.all(np.abs(outs[1] - ref) <= bnd), (N, direction, ratio)
        assert np.all(outs[1][N:] == 0)                 # identity padding, zero right-hand side in the padding


def test_trsv_rejections_launch_nothing(engine):
    s = _sms()
    buf = _dev(np.zeros(4 * T * T))
    p = buf.data_ptr()
    n0 = engine.launch_count()
    for sched, direction, args in ((2, 0, [p, T, p, p, p, T]), (0, 2, [p, T, p, p, p, T]), (0, 0, [p, T, p, p, p]),
                                   (0, 0, [p, T, p, p, p, 100]), (0, 0, [p, 129, p, p, p, T]), (1, 0, [p + 8, T, p, p, p, T]),
                                   (0, 1, [0, T, p, p, p, T]), (1, 1, [p, T, p, p, p, (4 * s + 1) * T])):
        with pytest.raises(ValueError):
            engine.trsv_tiles(sched, direction, args)
    assert engine.launch_count() == n0


# ---- GPA kernels -----------------------------------------------------------------------------------------------------

def _trmv_run(engine, which, Fh, ld, x):
    Npad = x.shape[0]
    dF, dx, do = _dev(Fh), _dev(_tail(x, T)), _dev(np.full(Npad + T, POISON))
    n0 = engine.launch_count()
    engine.gpa_kernels(which, [dF.data_ptr(), ld, dx.data_ptr(), do.data_ptr(), Npad])
    assert engine.launch_count() == n0 + 1
    out = _host(do)
    assert np.array_equal(_raw(out[Npad:]), _raw(np.full(T, POISON)))
    assert np.array_equal(_raw(_host(dF)), _raw(Fh))
    return out[:Npad]


@pytest.mark.parametrize("Npad,ld", [(128, 128), (1024, 1024 + 128), (4224, 4224)])
def test_trmv_exact_bitwise_upper_triangle_poisoned(engine, Npad, ld):
    rng = np.random.default_rng(Npad)
    m = vm.trmv_read_mask(Npad, ld)
    Fh = np.where(m, vm.dyadic(rng, (Npad, ld)), POISON)
    x = rng.integers(-4, 5, Npad).astype(np.float64)
    for which, model in ((0, vm.trmv), (1, vm.trmv_t)):
        got = _trmv_run(engine, which, Fh, ld, x)
        want = model(Fh, x)
        bad = _bits(got) != _bits(want)
        assert not bad.any(), (which, Npad, int(bad.sum()), np.argwhere(bad)[0])


def test_trmv_real_factor_within_bound(engine):
    _need_longdouble()
    Lr, rng = _real_factor(2000, seed=7)
    Npad = 2048
    L = np.eye(Npad)
    L[:2000, :2000] = Lr
    Fh = np.where(vm.trmv_read_mask(Npad, Npad), L, POISON)
    x = np.zeros(Npad)
    x[:2000] = rng.standard_normal(2000)
    for which, model, bound in ((0, vm.trmv, vm.trmv_bound), (1, vm.trmv_t, vm.trmv_t_bound)):
        got = _trmv_run(engine, which, Fh, Npad, x)
        ref, bnd = model(Fh, x, np.longdouble), bound(Fh, x)
        err = np.abs(got - ref)
        ratio = float(np.max(err / np.where(bnd > 0, bnd, np.inf)))
        print("RATIO trmv which=%d max|err|/bound = %.3e" % (which, ratio))
        assert np.all(err <= bnd), ratio
        assert np.array_equal(_raw(got), _raw(_trmv_run(engine, which, Fh, Npad, x)))


def _scan_run(engine, G, DinvT, u, v, F0, Z0):
    Npad = u.shape[0]
    ld = G.shape[1]
    dG, dD, du, dv, dF, dZ = _dev(G), _dev(DinvT), _dev(_tail(u, T)), _dev(_tail(v, T)), _dev(F0), _dev(Z0)
    n0 = engine.launch_count()
    engine.gpa_kernels(2, [dG.data_ptr(), ld, dD.data_ptr(), du.data_ptr(), dv.data_ptr(), dF.data_ptr(), dZ.data_ptr(), Npad])
    assert engine.launch_count() == n0 + 1
    assert np.array_equal(_raw(_host(dG)), _raw(G)) and np.array_equal(_raw(_host(dD)), _raw(DinvT))
    return _host(dF), _host(dZ)


def _scan_inputs(rng, Npad, ld, exact):
    fw, dr = vm.scan_masks(Npad, ld)
    if exact:
        G = np.where(fw, vm.dyadic(rng, (Npad, ld)), POISON)
        D = np.where(dr, vm.dyadic(rng, (Npad, T)), POISON)
        u, v = (rng.integers(-4, 5, Npad).astype(np.float64) for _ in range(2))
    else:
        G = np.where(fw, rng.standard_normal((Npad, ld)) / np.sqrt(Npad), POISON)
        D = np.where(dr, rng.standard_normal((Npad, T)), POISON)
        u, v = rng.standard_normal(Npad), rng.standard_normal(Npad)
    return fw, G, D, u, v


# Npad = 4224: rows b = 127, 128, 2175, 2176, 2177, 4223 have 4097, 4096, 2049, 2048, 2047 and 1 entries (b = 127, 2175,
# 2177 lie inside a tile, b != tb0); rows longer than 2048 carry sums across chunks
@pytest.mark.parametrize("Npad,ld", [(4224, 4224), (384, 384 + 256)])
def test_gpa_scan_exact_bitwise_regions_and_poison(engine, Npad, ld):
    rng = np.random.default_rng(Npad)
    fw, G, D, u, v = _scan_inputs(rng, Npad, ld, exact=True)
    # F: the lower triangle and diagonal tiles (where the engine keeps L) and every column past Npad must stay as they are
    F0 = np.full((Npad, ld), POISON)
    F0[~fw] = vm.dyadic(rng, (Npad, ld))[~fw]
    Z0 = np.full((Npad, T), POISON)                    # ZdT starts as NaN everywhere: the entries left of b must be zeroed
    Fo, Zo = _scan_run(engine, G, D, u, v, F0, Z0)
    Zf, ZdT = vm.gpa_scan(G, D, u, v)
    assert np.array_equal(_raw(Fo[~fw]), _raw(F0[~fw]))
    bad = _bits(Fo[:, :Npad][fw[:, :Npad]]) != _bits(Zf[fw[:, :Npad]])
    assert not bad.any(), int(bad.sum())
    bad = _bits(Zo) != _bits(ZdT)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[0])
    b = np.arange(Npad)
    left = np.arange(T)[None, :] < (b % T)[:, None]
    assert np.array_equal(_raw(Zo[left]), np.zeros(int(left.sum()), np.uint64))        # +0.0, not NaN, not -0.0


def test_gpa_scan_gaussian_within_bound_and_repeatable(engine):
    _need_longdouble()
    Npad = 4224
    rng = np.random.default_rng(17)
    fw, G, D, u, v = _scan_inputs(rng, Npad, Npad, exact=False)
    F0, Z0 = np.full((Npad, Npad), POISON), np.full((Npad, T), POISON)
    Fo, Zo = _scan_run(engine, G, D, u, v, F0, Z0)
    Zf, ZdT = vm.gpa_scan(G, D, u, v, np.longdouble)
    bf, bd = vm.gpa_scan_bound(G, D, u, v)
    ef, ed = np.abs(Fo[fw] - Zf[fw]), np.abs(Zo - ZdT)
    ratio = max(float(np.max(ef / bf[fw])), float(np.max(ed / np.where(bd > 0, bd, np.inf))))
    print("RATIO gpa_scan max|err|/bound = %.3e" % ratio)
    assert np.all(ef <= bf[fw]) and np.all(ed <= bd), ratio
    Fo2, Zo2 = _scan_run(engine, G, D, u, v, F0, Z0)
    assert np.array_equal(_raw(Fo2), _raw(Fo)) and np.array_equal(_raw(Zo2), _raw(Zo))


def test_gpa_rejections_launch_nothing(engine):
    buf = _dev(np.zeros(T * T))
    p = buf.data_ptr()
    n0 = engine.launch_count()
    for which, args in ((3, [p, T, p, p, T]), (0, [p, T, p, p]), (0, [p, T, p, p, 100]), (1, [p, 64, p, p, T]),
                        (2, [p, T, p, p, p, p, p]), (2, [p, T, p, 0, p, p, p, T])):
        with pytest.raises(ValueError):
            engine.gpa_kernels(which, args)
    assert engine.launch_count() == n0


# ---- fixed-order reductions -------------------------------------------------------------------------------------------

NS = [0, 1, 255, 256, 257, 1023, 1024, 1025, 3 * 1024 + 7, 10 ** 6]


def _reduce(engine, which, arrays, scalars, out_len):
    """arrays: host arrays (uploaded); scalars: ints placed by position; returns the out buffer (out_len + 1 entries, the
    last one a POISON sentinel that must come back unchanged)"""
    devs = [_dev(a) for a in arrays]
    do = _dev(np.full(out_len + 1, POISON))
    it = iter(devs)
    args = [next(it).data_ptr() if s is None else s for s in scalars] + [do.data_ptr()]
    n0 = engine.launch_count()
    engine.row_reductions(which, args)
    launched = engine.launch_count() - n0
    out = _host(do)
    assert np.array_equal(_raw(out[out_len:]), _raw(np.full(1, POISON)))
    for d, a in zip(devs, arrays):
        assert np.array_equal(_raw(_host(d)), _raw(a))
    return out[:out_len], launched


def _rows(n):
    return 3 if n >= 10 ** 6 else 5


@pytest.mark.parametrize("n", NS)
def test_dot_sum_exact_bitwise_tail_poisoned(engine, n):
    rng = np.random.default_rng(n)
    a, b = _tail(vm.dyadic(rng, n), 1031), _tail(vm.dyadic(rng, n), 1031)
    out, k = _reduce(engine, 0, [a, b], [None, None, n], 1)
    assert k == 1 and _bits(out[0]) == _bits(np.float64(vm.dot(a, b, n))), (n, out[0], vm.dot(a, b, n))
    out, k = _reduce(engine, 1, [a], [None, n], 1)
    assert k == 1 and _bits(out[0]) == _bits(np.float64(vm.vsum(a, n))), (n, out[0], vm.vsum(a, n))


@pytest.mark.parametrize("n", NS)
def test_row_reductions_exact_bitwise_row_tails_poisoned(engine, n):
    rng = np.random.default_rng(n + 1)
    M, ld = _rows(n), n + 37
    K = np.full((M, ld), POISON)
    K[:, :n] = vm.dyadic(rng, (M, n))
    B = np.full((M, ld), POISON)
    B[:, :n] = vm.dyadic(rng, (M, n))
    alpha = _tail(vm.dyadic(rng, n), 64)
    kd = _tail(vm.dyadic(rng, M) * 64, 3)
    out, k = _reduce(engine, 2, [K, alpha], [None, ld, None, M, n], M)
    assert k == 1 and np.array_equal(_bits(out), _bits(vm.rowdot(K, alpha, M, n))), n
    out, k = _reduce(engine, 3, [K, kd], [None, ld, None, M, n], M)
    assert k == 1 and np.array_equal(_bits(out), _bits(vm.rowvar(K, kd, M, n))), n
    out, k = _reduce(engine, 4, [K, B], [None, None, ld, M, n], M)
    assert k == 1 and np.array_equal(_bits(out), _bits(vm.rowdot2(K, B, M, n))), n


@pytest.mark.parametrize("n", [257, 1025, 3 * 1024 + 7, 10 ** 6])
def test_reductions_gaussian_within_bound_and_repeatable(engine, n):
    _need_longdouble()
    rng = np.random.default_rng(n + 2)
    a, b = _tail(rng.standard_normal(n), 8), _tail(rng.standard_normal(n), 8)
    M, ld = _rows(n), n + 5
    K = np.full((M, ld), POISON)
    K[:, :n] = rng.standard_normal((M, n))
    B = np.full((M, ld), POISON)
    B[:, :n] = rng.standard_normal((M, n))
    kd = _tail(rng.standard_normal(M) + n, 1)
    cases = [("dot", 0, [a, b], [None, None, n], 1, vm.dot(a, b, n, np.longdouble), vm.dot_bound(a, b, n)),
             ("sum", 1, [a], [None, n], 1, vm.vsum(a, n, np.longdouble), vm.vsum_bound(a, n)),
             ("rowdot", 2, [K, a], [None, ld, None, M, n], M, vm.rowdot(K, a, M, n, np.longdouble), vm.rowdot_bound(K, a, M, n)),
             ("rowvar", 3, [K, kd], [None, ld, None, M, n], M, vm.rowvar(K, kd, M, n, np.longdouble), vm.rowvar_bound(K, kd, M, n)),
             ("rowdot2", 4, [K, B], [None, None, ld, M, n], M, vm.rowdot2(K, B, M, n, np.longdouble), vm.rowdot2_bound(K, B, M, n))]
    for name, which, arrays, scalars, m, ref, bnd in cases:
        out, _ = _reduce(engine, which, arrays, scalars, m)
        err = np.abs(out - ref)
        ratio = float(np.max(err / bnd))
        print("RATIO %s n=%d max|err|/bound = %.3e" % (name, n, ratio))
        assert np.all(err <= bnd), (name, n, ratio)
        again, _ = _reduce(engine, which, arrays, scalars, m)
        assert np.array_equal(_raw(again), _raw(out)), name


def test_reductions_empty_rows_and_rejections(engine):
    K = _dev(np.zeros(64))
    p = K.data_ptr()
    n0 = engine.launch_count()
    for which in (2, 3, 4):
        engine.row_reductions(which, [p, 8, p, 0, 8, p] if which != 4 else [p, p, 8, 0, 8, p])    # M = 0: nothing to do
    assert engine.launch_count() == n0
    for which, args in ((5, [p, p, 8, p]), (0, [p, p, 8]), (0, [p, p, -1, p]), (1, [0, 8, p]), (2, [p, 7, p, 2, 8, p]),
                        (3, [p, 8, 0, 2, 8, p]), (4, [p, 0, 8, 2, 8, p]), (4, [p, p, 8, -1, 8, p])):
        with pytest.raises(ValueError):
            engine.row_reductions(which, args)
    assert engine.launch_count() == n0
