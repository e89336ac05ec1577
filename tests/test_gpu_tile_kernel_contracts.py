"""GPU: the three kernels that carry the O(N^3) work, tested directly against their contracts.

* NT GEMM (csrc/gemm_nt.cu) through gpb200_gemm_nt_desc, both loaders, against the descriptor model tests/gemm_model.py.
  Exact cases use operands k * 2^-8 (|k| <= 256) and alpha, beta in {1, -1, 0.5, -0.75, 0}: every product, partial sum
  (K <= 8192) and alpha * acc + beta * C is exact in FP64, so device and model agree bit for bit whatever the summation
  order.  Every element the model says is not read holds a NaN, so a read outside the declared k range or of a main-buffer
  diagonal tile that `sub` replaces shows up; every element outside the written region holds a NaN with its own payload
  that must come back bit-identical; with beta = 0 the written region starts as NaN, because C must not be read.
* Grouped tile GEMM (csrc/fsa.cu) through gpb200_fsa_gemm_items, bitwise against the same exact model and against the NT
  GEMM (both issue the same MMAs in the same order).
* Diagonal-tile leaf (csrc/potrf_base.cu) through gpb200_potrf_tiles, both entry points, against an extended-precision
  Cholesky: backward-error bounds, clean inverse triangles, logd, untouched regions, peer copies and the info word.

The file sorts after test_gpu_gpa.py and test_gpu_launch_count.py on purpose: torch.profiler records no device activity
in a session started about a minute or more after the process's first profiling session, so this file's run time must
not fall between the two."""
import numpy as np
import pytest

import gemm_model as gm
from gemm_model import KHI_M, KHI_N, KLO_M, KLO_N, LOWER_ONLY, SKIP_FIRST, Desc, Operand

pytestmark = pytest.mark.gpu

T = 128
U = 2.0 ** -53
POISON = np.array([0x7FF8_DEAD_0000_0001], dtype=np.uint64).view(np.float64)[0]   # "never read, never written"
ALPHAS = (1.0, -1.0, 0.5, -0.75)


def _bits(a):
    a = np.where(a == 0, 0.0, a)                 # +0 and -0 are the same result of an exact sum
    return np.ascontiguousarray(a).view(np.uint64)


def _exact(rng, shape):
    return rng.integers(-256, 257, size=shape).astype(np.float64) / 256.0


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


# ---- NT GEMM through the flat descriptor ----------------------------------------------------------------------------

def _flat_desc(d, dev, nomap=()):
    f = [d.flags, d.M, d.N, d.K, d.batch, d.zstep, d.m_lim, d.n_lim, d.k_lim, d.klo_off, d.bm_mod, d.bm_rem, d.bn_mod,
         d.bn_rem, d.bm_div, d.bm_off, d.bn_div, d.bn_off, len(d.peers), d.A.row0, d.A.col0, d.B.row0, d.B.col0,
         d.c_row0, d.c_col0, d.ct_row0, d.ct_col0]

    def buf(name):
        if name is None:
            return [0, 0, 0, 0]
        t = dev[name]
        rows, cols = t.shape
        if name in nomap:
            rows = cols = 0
        return [t.data_ptr(), rows, cols, t.stride(0)]

    for name in (d.A.buf, d.A.sub, d.B.buf, d.B.sub, d.C, d.Ct):
        f += buf(name)
    for q in range(7):
        f += buf(d.peers[q] if q < len(d.peers) else None)
    assert len(f) == 79
    return np.array(f, dtype=np.int64)


def _initial(d, shapes, fill):
    """Buffers the launch may read hold `fill` values, the rest POISON; with beta = 0 the written region holds NaN."""
    read, written = gm.run(d, {k: np.zeros(s) for k, s in shapes.items()})
    init = {}
    for k, s in shapes.items():
        a = np.full(s, POISON)
        a[written[k]] = np.nan
        v = fill(s)
        a[read[k]] = v[read[k]]
        init[k] = a
    return init


def _run_exact(engine, d, shapes, impl, seed=0, nomap=()):
    rng = np.random.default_rng(seed)
    init = _initial(d, shapes, lambda s: _exact(rng, s))
    want = {k: v.copy() for k, v in init.items()}
    gm.run(d, want)
    dev = {k: _dev(v) for k, v in init.items()}
    n0 = engine.launch_count()
    engine.gemm_nt_desc(impl, _flat_desc(d, dev, nomap), d.alpha, d.beta)
    assert engine.launch_count() == n0 + 1
    for k in shapes:
        got = _host(dev[k])
        bad = _bits(got) != _bits(want[k])
        assert not bad.any(), "%s: %d elements differ, first at %s" % (k, bad.sum(), np.argwhere(bad)[0])
    return want


def _sq(n):
    return (n, n)


# every flag alone; origins inside larger buffers, alpha / beta from the exact set
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("flags", [0, LOWER_ONLY, KLO_M, KHI_M, KHI_N, SKIP_FIRST, KLO_N])
def test_gemm_each_flag_alone(engine, impl, flags):
    for alpha, beta in ((-0.75, 0.5), (1.0, 0.0)):
        d = Desc(Operand("A", None, 128, 16), Operand("B", None, 256, 32), "C", c_row0=128, c_col0=256,
                 M=384, N=384, K=384, alpha=alpha, beta=beta, flags=flags)
        _run_exact(engine, d, dict(A=(640, 512), B=(768, 448), C=(640, 768)), impl, seed=flags)


def _engine_cases():
    Np = 640
    sq = dict(G=_sq(Np), F=_sq(Np), Dinv=(Np, T), DinvT=(Np, T))
    # panel_trsm_leaf (gpb200.cu): F[r0.., p..) = G[r0.., p..) W_pp'
    yield "panel_trsm_leaf", Desc(Operand("G", None, 256, 128), Operand("Dinv", None, 128, 0), "F", c_row0=256,
                                  c_col0=128, M=384, N=T, K=T), sq
    # schur_update (gpb200.cu) and its look-ahead remainder (chol_panel)
    for extra in (0, SKIP_FIRST):
        yield "schur_update", Desc(Operand("F", None, 256, 0), Operand("F", None, 256, 0), "G", c_row0=256, c_col0=256,
                                   M=384, N=256, K=256, alpha=-1.0, beta=1.0, flags=LOWER_ONLY | extra), sq
    # merge_inverse (gpb200.cu) at Npad = 896: both launches of level s = 128 (batch 4, the last problem skipped) and of
    # s = 256 (batch 2, the second problem clipped to one tile)
    Nm = 896
    sqm = dict(G=_sq(Nm), F=_sq(Nm), Dinv=(Nm, T), DinvT=(Nm, T))
    for s in (128, 256):
        batch, lim, n2 = (Nm + 2 * s - 1) // (2 * s), Nm - s, min(Nm - s, s)
        yield "merge_inverse_T", Desc(Operand("G", "DinvT", 0, 0), Operand("F", None, s, 0), "F", c_row0=0, c_col0=s,
                                      M=s, N=n2, K=s, flags=KLO_M, batch=batch, zstep=2 * s, n_lim=lim), sqm
        yield "merge_inverse_W21", Desc(Operand("G", "Dinv", s, s), Operand("F", None, 0, s), "G", c_row0=s, c_col0=0,
                                        Ct="G", ct_row0=0, ct_col0=s, M=n2, N=s, K=n2, alpha=-1.0, flags=KHI_M,
                                        batch=batch, zstep=2 * s, m_lim=lim, k_lim=lim), sqm
    # inverse_from_factor (gpb200.cu): W'W, A = B = G with the DinvT tiles on the diagonal
    yield "inverse_from_factor", Desc(Operand("G", "DinvT"), Operand("G", "DinvT"), "G", M=Np, N=Np, K=Np,
                                      flags=LOWER_ONLY | KLO_M), sq
    # GPA product (gpb200_gpa_grad, gpb200.cu): B's diagonal tiles from a second sub buffer
    yield "gpa_product", Desc(Operand("G", "DinvT"), Operand("F", "ZdT"), "G", M=Np, N=Np, K=Np, alpha=-1.0,
                              flags=LOWER_ONLY | KLO_M), dict(sq, ZdT=(Np, T))
    # rand (rand_from_cov, gpb200.cu): out = Z L'
    yield "rand", Desc(Operand("Z"), Operand("F"), "O", M=256, N=Np, K=Np, flags=KHI_N), dict(Z=(256, Np), F=_sq(Np),
                                                                                               O=(256, Np))
    # rank update of a symmetric block (gpb200_fitc_factorize, fitc_engine.cu): C += B B', lower trapezoid
    yield "rank_update", Desc(Operand("B"), Operand("B"), "C", M=512, N=512, K=384, beta=1.0, flags=LOWER_ONLY), \
        dict(B=(512, 384), C=_sq(512))
    # inverse_dist (gpb200.cu): the two merge launches of level s = 256 split over 2 ranks (filtered grids, batch 2,
    # the second problem clipped)
    for me in range(2):
        yield "inverse_dist_T", Desc(Operand("G", "DinvT"), Operand("F", None, 256, 0), "F", c_row0=0, c_col0=256,
                                     M=256, N=256, K=256, flags=KLO_M, bm_mod=2, bm_rem=me, batch=2, zstep=512,
                                     n_lim=Nm - 256), sqm
        yield "inverse_dist_W21", Desc(Operand("G", "Dinv", 256, 256), Operand("F", None, 0, 256), "G", c_row0=256,
                                       c_col0=0, Ct="G", ct_row0=0, ct_col0=256, M=256, N=256, K=256, alpha=-1.0,
                                       flags=KHI_M, bn_mod=2, bn_rem=me, batch=2, zstep=512, m_lim=Nm - 256,
                                       k_lim=Nm - 256), sqm
    for me in range(3):
        # inverse_dist: W'W on the owned tile rows (compact grid, batch 1)
        yield "inverse_dist_WtW", Desc(Operand("G", "DinvT"), Operand("G", "DinvT"), "G", M=Np, N=Np, K=Np,
                                       flags=LOWER_ONLY | KLO_M, bm_mod=3, bm_rem=me), sq
    # shard_impl.cuh: own_rows_filter (l. 402) on the leaf TRSM (l. 414), the narrow Schur update (l. 523), the TRTRI
    # panel with its transposed store into G (l. 651, ldc != ldct) and the LAUUM part (l. 711)
    for rank, rb in ((0, 1), (1, 2)):
        own = dict(bm_mod=2, bm_rem=rank, bm_div=rb, bm_off=1)
        yield "shard_trsm", Desc(Operand("G", None, 128, 0), Operand("Dinv"), "G", c_row0=128, c_col0=0,
                                 M=512, N=T, K=T, **own), dict(G=_sq(Np), Dinv=(Np, T))
        yield "shard_narrow", Desc(Operand("P", None, 128, 0), Operand("P", None, 128, 0), "G", c_row0=128, c_col0=128,
                                   M=512, N=256, K=256, alpha=-1.0, beta=1.0, flags=LOWER_ONLY, **own), \
            dict(P=(Np, 256), G=_sq(Np))
        yield "shard_lauum", Desc(Operand("G", "DinvT", 128, 128), Operand("XR", None, 0, 128), "G", c_row0=128,
                                  c_col0=128, M=512, N=256, K=512, flags=LOWER_ONLY | KLO_M, **own), \
            dict(G=_sq(Np), DinvT=(Np, T), XR=(256, Np))
    yield "shard_trtri", Desc(Operand("S", None, 384, 0), Operand("G", "DinvT", 128, 128), "P", c_row0=384, c_col0=0,
                              Ct="G", ct_row0=128, ct_col0=384, M=256, N=256, K=256, alpha=-1.0, flags=KLO_N), \
        dict(S=(Np, 256), G=_sq(Np), DinvT=(Np, T), P=(Np, 256))


_CASES = list(_engine_cases())


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("case", range(len(_CASES)), ids=["%s-%d" % (c[0], i) for i, c in enumerate(_CASES)])
def test_gemm_engine_descriptors_exact(engine, impl, case):
    _, d, shapes = _CASES[case]
    _run_exact(engine, d, shapes, impl, seed=case)


@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_rasterisation_wraps_partial_groups(engine, impl):
    # tm = 21: GROUP_M 16 leaves a group of 5, GM_TRI 4 a group of 1
    for flags in (0, KLO_M, LOWER_ONLY, LOWER_ONLY | KLO_M):
        N = 3 * T if not flags & LOWER_ONLY else 21 * T
        K = 48 if not flags & KLO_M else 21 * T
        d = Desc(Operand("A"), Operand("B"), "C", M=21 * T, N=N, K=K, alpha=0.5, beta=-1.0, flags=flags)
        _run_exact(engine, d, dict(A=(21 * T, K), B=(N, K), C=(21 * T, N)), impl, seed=flags)


@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_short_k_ranges(engine, impl):
    for nk in (1, 2, 5, 6, 11):                               # fewer, equal and more k-steps than pipeline stages
        d = Desc(Operand("A", None, 0, 32), Operand("B", None, 0, 32), "C", M=256, N=256, K=16 * nk, alpha=-1.0)
        _run_exact(engine, d, dict(A=(256, 256), B=(256, 256), C=(256, 256)), impl, seed=nk)
    # KLO_M: tile row 1 gets 0, 1, 5 and 6 k-steps (row 0 eight more), walked downwards
    for K, klo_off in ((128, 0), (144, 0), (208, 0), (240, 16)):
        d = Desc(Operand("A"), Operand("B"), "C", M=256, N=384, K=K, klo_off=klo_off, alpha=-0.75, beta=1.0, flags=KLO_M)
        _run_exact(engine, d, dict(A=(256, 256), B=(384, 256), C=(256, 384)), impl, seed=K)


@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_batches_clip_and_skip(engine, impl):
    # z = 2 clipped to one tile row / column / k tile, z = 3 skipped (m_lim - 3 zstep < 0)
    for lim in ("m_lim", "n_lim", "k_lim"):
        d = Desc(Operand("A", None, 0, 0), Operand("B", None, 0, 0), "C", M=256, N=256, K=256, beta=0.5,
                 batch=4, zstep=256, **{lim: 640})
        _run_exact(engine, d, dict(A=(1024, 1024), B=(1024, 1024), C=(1024, 1024)), impl, seed=len(lim))


@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_transposed_copy_and_peers(engine, impl):
    d = Desc(Operand("A"), Operand("B"), "C", c_row0=128, c_col0=0, Ct="Ct", ct_row0=0, ct_col0=256, M=384, N=256,
             K=96, alpha=-1.0, beta=0.5)
    _run_exact(engine, d, dict(A=(384, 96), B=(256, 96), C=(512, 256), Ct=(384, 768)), impl)
    for n_peer in (1, 2, 3):
        peers = tuple("P%d" % q for q in range(n_peer))
        d = Desc(Operand("A"), Operand("B"), "C", c_row0=128, c_col0=128, M=256, N=384, K=160, alpha=0.5, beta=-0.75,
                 peers=peers)
        shapes = dict(A=(256, 160), B=(384, 160), C=(384, 512), **{p: (384, 512) for p in peers})
        want = _run_exact(engine, d, shapes, impl, seed=n_peer)
        w = gm.run(d, {k: np.zeros(s) for k, s in shapes.items()})[1]["C"]
        for p in peers:
            assert np.array_equal(_bits(want[p][w]), _bits(want["C"][w]))


def test_gemm_rejections_launch_nothing(engine):
    dev = dict(A=_dev(np.zeros((256, 256))), B=_dev(np.zeros((256, 256))), C=_dev(np.zeros((256, 256))),
               Ct=_dev(np.zeros((256, 256))), P0=_dev(np.zeros((256, 256))), S=_dev(np.zeros((256, 128))),
               O=_dev(np.zeros((256, 255))))
    base = dict(M=256, N=256, K=256)
    bad = [(0, Desc(Operand("A"), Operand("B"), "C", flags=LOWER_ONLY, peers=("P0",), **base), ()),
           (1, Desc(Operand("A"), Operand("B"), "C", flags=LOWER_ONLY, peers=("P0",), **base), ()),
           (0, Desc(Operand("A"), Operand("B"), "C", flags=LOWER_ONLY, Ct="Ct", **base), ()),
           (1, Desc(Operand("A"), Operand("B"), "C", flags=LOWER_ONLY, Ct="Ct", **base), ()),
           (0, Desc(Operand("A"), Operand("B"), "C", M=200, N=256, K=256), ()),
           (1, Desc(Operand("A"), Operand("B"), "C", M=256, N=256, K=24), ()),
           (1, Desc(Operand("A"), Operand("B"), "O", M=256, N=128, K=128), ()),      # odd ldc
           (0, Desc(Operand("A", "S"), Operand("B"), "C", **base), ("S",)),            # TMA kernel, sub without a map
           (0, Desc(Operand("A"), Operand("B", "S"), "C", **base), ("S",))]
    for impl, d, nomap in bad:
        n0 = engine.launch_count()
        with pytest.raises(ValueError):
            engine.gemm_nt_desc(impl, _flat_desc(d, dev, nomap), 1.0, 0.0)
        assert engine.launch_count() == n0
    # the simple kernel reads a sub buffer through its pointer: the same launch is valid there
    d = Desc(Operand("A", "S"), Operand("B"), "C", **base)
    _run_exact(engine, d, dict(A=(256, 256), S=(256, 128), B=(256, 256), C=(256, 256)), 1, nomap=("S",))


def _run_gauss(engine, d, shapes, seed):
    rng = np.random.default_rng(seed)
    init = _initial(d, shapes, lambda s: rng.standard_normal(s))
    want = {k: v.astype(np.longdouble) for k, v in init.items()}
    gm.run(d, want, acc_dtype=np.longdouble)
    absd = Desc(**{**d.__dict__, "alpha": abs(d.alpha), "beta": abs(d.beta)})
    mag = {k: np.where(np.isnan(v), 0.0, np.abs(v)).astype(np.longdouble) for k, v in init.items()}
    gm.run(absd, mag, acc_dtype=np.longdouble)
    nk = np.zeros(shapes[d.C])
    for t in gm.tiles(d):
        zo = t.z * d.zstep
        nk[d.c_row0 + zo + t.bm * T:d.c_row0 + zo + (t.bm + 1) * T, d.c_col0 + zo + t.bn * T:d.c_col0 + zo + (t.bn + 1) * T] \
            = max(t.khi - t.klo, 0)
    written = gm.run(d, {k: np.zeros(s) for k, s in shapes.items()})[1][d.C]
    outs = []
    for impl in (0, 1):
        dev = {k: _dev(v) for k, v in init.items()}
        engine.gemm_nt_desc(impl, _flat_desc(d, dev), d.alpha, d.beta)
        outs.append(_host(dev[d.C]))
    assert np.array_equal(_bits(outs[0]), _bits(outs[1])), "TMA and simple loaders differ"
    got = outs[0]
    err = np.abs(got[written].astype(np.longdouble) - want[d.C][written])
    bound = (nk[written] + 2) * U * mag[d.C][written]
    assert (err <= bound).all(), float(np.max(err / np.maximum(bound, 1e-300)))
    assert np.array_equal(_bits(got[~written]), _bits(init[d.C][~written]))


@pytest.mark.parametrize("flags", [0, LOWER_ONLY, KLO_M | LOWER_ONLY, KHI_M, KHI_N | SKIP_FIRST, KLO_N])
def test_gemm_rounding_gaussian_operands(engine, flags):
    d = Desc(Operand("A", None, 0, 64), Operand("B", None, 128, 0), "C", M=512, N=384, K=512, alpha=-0.7, beta=1.3,
             flags=flags)
    _run_gauss(engine, d, dict(A=(512, 640), B=(512, 512), C=(512, 384)), seed=flags)
    d = Desc(Operand("A", "S"), Operand("A", "S"), "C", M=384, N=384, K=384, alpha=1.1, flags=flags | LOWER_ONLY)
    _run_gauss(engine, d, dict(A=(384, 384), S=(384, 128), C=(384, 384)), seed=flags + 100)


# ---- grouped tile GEMM ----------------------------------------------------------------------------------------------

def test_fsa_gemm_items_exact(engine):
    rng = np.random.default_rng(5)
    src = {128: _exact(rng, (256, 128)), 384: _exact(rng, (384, 384)), 512: _exact(rng, (512, 512)),
           2048: _exact(rng, (256, 2048))}
    outs = {128: (16 * T, 128), 384: (384, 384), 512: (512, 512)}
    out_tiles = [(ld, r, c) for ld, (R, C) in outs.items() for r in range(0, R, T) for c in range(0, C, T)]
    rng.shuffle(out_tiles)
    init = {ld: np.full(s, POISON) for ld, s in outs.items()}
    plan = []
    for i, (ldc, r, c) in enumerate(out_tiles):
        K = (0, 16, 32, 48, 2048)[i % 5]
        lower, beta, alpha = i % 2, (0.0, 1.0, -0.75)[i % 3], ALPHAS[i % 4]
        ld = 2048 if K == 2048 else (128, 384, 512)[(i // 5) % 3]
        S = src[ld]
        ra = 0 if i % 3 == 0 else int(rng.integers(0, S.shape[0] // T)) * T     # every third item shares A rows 0
        rb = int(rng.integers(0, S.shape[0] // T)) * T
        k0 = int(rng.integers(0, (S.shape[1] - K) // 16 + 1)) * 16
        init[ldc][r:r + T, c:c + T] = _exact(rng, (T, T)) if beta != 0.0 else np.nan
        plan.append((ldc, r, c, ld, ra, rb, k0, K, lower, alpha, beta))
    want = {k: v.copy() for k, v in init.items()}
    for ldc, r, c, ld, ra, rb, k0, K, lower, alpha, beta in plan:
        acc = src[ld][ra:ra + T, k0:k0 + K] @ src[ld][rb:rb + T, k0:k0 + K].T
        v = alpha * acc + (beta * want[ldc][r:r + T, c:c + T] if beta != 0.0 else 0.0)
        m = np.tri(T, dtype=bool) if lower else np.ones((T, T), bool)
        want[ldc][r:r + T, c:c + T][m] = v[m]
    dsrc = {k: _dev(v) for k, v in src.items()}
    dout = {k: _dev(v) for k, v in init.items()}
    items = [[dout[ldc].data_ptr() + 8 * (r * ldc + c), dsrc[ld].data_ptr() + 8 * (ra * ld + k0),
              dsrc[ld].data_ptr() + 8 * (rb * ld + k0), ldc, ld, ld, K, lower]
             for ldc, r, c, ld, ra, rb, k0, K, lower, alpha, beta in plan]
    ab = [(p[9], p[10]) for p in plan]
    n0 = engine.launch_count()
    engine.fsa_gemm_items(np.array(items), np.array(ab))
    assert engine.launch_count() == n0 + 1
    for k in outs:
        got = _host(dout[k])
        bad = _bits(got) != _bits(want[k])
        assert not bad.any(), "ldc %d: %d elements differ, first at %s" % (k, bad.sum(), np.argwhere(bad)[0])
    for k in src:
        assert np.array_equal(_host(dsrc[k]), src[k])


def test_fsa_gemm_matches_gemm_nt_bitwise(engine):
    rng = np.random.default_rng(9)
    for K in (16, 48, 512):
        A, B, C0 = rng.standard_normal((T, K)), rng.standard_normal((T, K)), rng.standard_normal((T, T))
        dA, dB = _dev(A), _dev(B)
        c1, c2 = _dev(C0), _dev(C0)
        engine.fsa_gemm_items(np.array([[c1.data_ptr(), dA.data_ptr(), dB.data_ptr(), T, K, K, K, 0]]),
                              np.array([[-0.7, 1.3]]))
        d = Desc(Operand("A"), Operand("B"), "C", M=T, N=T, K=K, alpha=-0.7, beta=1.3)
        engine.gemm_nt_desc(0, _flat_desc(d, dict(A=dA, B=dB, C=c2)), d.alpha, d.beta)
        assert np.array_equal(_bits(_host(c1)), _bits(_host(c2))), K


# ---- diagonal-tile leaf ---------------------------------------------------------------------------------------------

def _need_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")


def _chol_ld(K):
    """lower Cholesky factor in long double (None past a non-positive pivot)"""
    n = K.shape[0]
    L = np.zeros((n, n), np.longdouble)
    A = np.tril(K).astype(np.longdouble)
    for j in range(n):
        d = A[j, j] - np.dot(L[j, :j], L[j, :j])
        if not d > 0:
            return None
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _tiles(rng):
    """well conditioned, SE Gram tiles (cond ~1e4 .. 1e12) and a tile with identity padding rows"""
    X = rng.standard_normal((T, T))
    out = [X @ X.T / T + np.eye(T)]
    x = np.sort(rng.uniform(0, 6, T))
    for nug in (1e-2, 1e-6, 1e-10):
        out.append(np.exp(-0.5 * (x[:, None] - x[None, :]) ** 2) + nug * np.eye(T))
    P = np.eye(T)
    P[:77, :77] = out[1][:77, :77]
    out.append(P)
    return out


def _check_leaf(K, L, W, WT, logd):
    Ll = L.astype(np.longdouble)
    Wl = W.astype(np.longdouble)
    n = T
    g = (n + 1) * U / (1 - (n + 1) * U)
    res = np.abs(np.tril(K).astype(np.longdouble) - np.tril(Ll @ Ll.T))
    assert (res <= g * np.tril(np.abs(Ll) @ np.abs(Ll).T)).all()
    # W is the block form of forward substitution on L W = I (column by column), so its right residual is small; the
    # left residual W L - I is bounded only through cond(L) (about 70 n u |W||L| on the cond-1e8 tile)
    r2 = np.abs(Ll @ Wl - np.eye(n))
    b2 = n * U * (np.abs(Ll) @ np.abs(Wl))
    assert (r2 <= 2 * b2).all(), float(np.max(r2 / (b2 + 1e-300)))
    assert np.array_equal(_bits(WT), _bits(np.ascontiguousarray(W.T)))
    assert np.array_equal(np.triu(W, 1).view(np.uint64), np.zeros((n, n), np.uint64))
    assert np.array_equal(np.tril(WT, -1).view(np.uint64), np.zeros((n, n), np.uint64))
    # logd = 2 log L_jj of the pivots the leaf stored, to a few ulp
    ref = 2 * np.log(np.diag(Ll))
    assert (np.abs(logd.astype(np.longdouble) - ref) <= 2 * np.spacing(np.abs(logd))).all()


def _mode0(engine, G, ntiles, p0, stride, n_peer=0):
    Np = G.shape[0]
    bufs = dict(G=G, F=np.full((Np, Np), POISON), Dinv=np.full((Np, T), POISON), DinvT=np.full((Np, T), POISON),
                logd=np.full((Np, 1), POISON))
    for q in range(n_peer):
        for k in ("F", "Dinv", "DinvT", "logd"):
            bufs["%s%d" % (k, q)] = bufs[k].copy()
    dev = {k: _dev(v) for k, v in bufs.items()}
    args = [dev["G"].data_ptr(), Np, dev["F"].data_ptr(), Np, dev["Dinv"].data_ptr(), dev["DinvT"].data_ptr(),
            dev["logd"].data_ptr(), p0, ntiles, stride, n_peer]
    for q in range(7):
        args += [dev["%s%d" % (k, q)].data_ptr() if q < n_peer else 0 for k in ("F", "Dinv", "DinvT", "logd")]
    info = engine.potrf_tiles(0, args)
    return info, {k: _host(v) for k, v in dev.items()}, bufs


def test_leaf_strided_tiles_bounds_and_untouched_regions(engine):
    _need_longdouble()
    rng = np.random.default_rng(1)
    tiles = _tiles(rng)
    stride, p0 = 256, 128
    Np = p0 + stride * (len(tiles) - 1) + T + 128
    G = np.full((Np, Np), POISON)
    for b, K in enumerate(tiles):
        p = p0 + b * stride
        G[p:p + T, p:p + T] = np.where(np.tri(T, dtype=bool), K, POISON)       # only the lower triangle is read
    info, out, init = _mode0(engine, G, len(tiles), p0, stride, n_peer=2)
    assert info == 2 ** 31 - 1
    touched = {k: np.zeros(v.shape, bool) for k, v in init.items()}
    for b, K in enumerate(tiles):
        p = p0 + b * stride
        L = out["F"][p:p + T, p:p + T]
        _check_leaf(K, np.tril(L), out["Dinv"][p:p + T], out["DinvT"][p:p + T], out["logd"][p:p + T, 0])
        touched["F"][p:p + T, p:p + T] = np.tri(T, dtype=bool)
        for k in ("Dinv", "DinvT", "logd"):
            touched[k][p:p + T] = True
    for k in ("G", "F", "Dinv", "DinvT", "logd"):
        m = ~touched.get(k, np.zeros(init[k].shape, bool))
        assert np.array_equal(_bits(out[k][m]), _bits(init[k][m])), k     # F's strict upper tile, G, padding rows
    for q in range(2):
        for k in ("F", "Dinv", "DinvT", "logd"):
            assert np.array_equal(_bits(out["%s%d" % (k, q)]), _bits(out[k])), (k, q)


def _mode1(engine, tiles, alias, info_base=0):
    items, dev = [], []
    for b, K in enumerate(tiles):
        ld = 384 if b % 2 else T
        G = np.full((T, ld), POISON)
        G[:, :T] = np.where(np.tri(T, dtype=bool), K, POISON)
        g = _dev(G)
        dv = g if alias else _dev(np.full((T, ld), POISON))
        dt, lg = _dev(np.full((T, ld), POISON)), _dev(np.full(T, POISON))
        dev.append((G, g, dv, dt, lg))
        items.append([g.data_ptr(), dv.data_ptr(), dt.data_ptr(), lg.data_ptr(), ld, info_base + 1000 * b])
    info = engine.potrf_tiles(1, items)
    return info, [(G, _host(g), _host(dv), _host(dt), _host(lg)) for G, g, dv, dt, lg in dev]


def test_leaf_pointer_table_matches_strided_and_allows_aliasing(engine):
    _need_longdouble()
    tiles = _tiles(np.random.default_rng(2))
    G = np.full((len(tiles) * T, len(tiles) * T), POISON)
    for b, K in enumerate(tiles):
        G[b * T:(b + 1) * T, b * T:(b + 1) * T] = np.tril(K)
    _, ref, _ = _mode0(engine, G, len(tiles), 0, T)
    runs = [_mode1(engine, tiles, alias) for alias in (False, True)]
    for alias, (info, res) in zip((False, True), runs):
        assert info == 2 ** 31 - 1
        for b, (G0, g, dv, dt, lg) in enumerate(res):
            s = slice(b * T, (b + 1) * T)
            assert np.array_equal(_bits(dv[:, :T]), _bits(ref["Dinv"][s])), (alias, b)
            assert np.array_equal(_bits(dt[:, :T]), _bits(ref["DinvT"][s])), (alias, b)
            assert np.array_equal(_bits(lg), _bits(ref["logd"][s, 0])), (alias, b)
            assert np.array_equal(_bits(dt[:, T:]), _bits(np.full((T, dt.shape[1] - T), POISON)))
            if not alias:
                assert np.array_equal(_bits(g), _bits(G0)), b          # G is only read


def _plant(K, j, value=None):
    """K with K[j, j] replaced so that pivot j is -1 (long-double Schur quadratic form of the leading block minus 1)"""
    K = K.copy()
    if value is None:
        L = _chol_ld(K[:j, :j])
        x = np.zeros(j, np.longdouble)                          # row j of the factor: L x = K[j, :j]
        for i in range(j):
            x[i] = (K[j, i] - np.dot(L[i, :i], x[:i])) / L[i, i]
        value = float(np.dot(x, x) - 1)
    K[j, j] = value
    return K


def test_leaf_info_is_the_first_non_positive_pivot(engine):
    _need_longdouble()
    base = _tiles(np.random.default_rng(3))[0]
    for j in (0, 1, 15, 16, 17, 63, 64, 127):
        K = _plant(base, j)
        info, _ = _mode1(engine, [K], False, info_base=40)
        assert info == 40 + j + 1, (j, info)
        G = np.zeros((3 * T, 3 * T))
        G[T:2 * T, T:2 * T] = np.tril(K)
        info, _, _ = _mode0(engine, G, 1, T, T)
        assert info == T + j + 1, (j, info)
    # two bad pivots: the first; bad tiles in one launch: the smallest
    info, _ = _mode1(engine, [_plant(_plant(base, 70), 20)], False)
    assert info == 21
    info, _ = _mode1(engine, [base, _plant(base, 90), _plant(base, 5)], False)   # info_base 0, 1000, 2000
    assert info == 1091
    G = np.zeros((4 * T, 4 * T))
    for b, K in enumerate((base, _plant(base, 90), _plant(base, 5))):
        G[b * T:(b + 1) * T, b * T:(b + 1) * T] = np.tril(K)
    info, _, _ = _mode0(engine, G, 3, 0, T)
    assert info == T + 91
    # an exact zero pivot and a NaN entry
    info, _ = _mode1(engine, [_plant(base, 0, 0.0)], False)
    assert info == 1
    K = base.copy()
    K[5, 3] = np.nan
    info, _ = _mode1(engine, [K], False)
    assert info == 6
