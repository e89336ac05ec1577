"""CPU (-m "not gpu"): the model of the TMA-staged SEIso kernels (tests/seiso_model.py) against itself and against long
double: the vectorised exact fma equals TwoProduct + one correctly rounded three-term sum, the fma-exact exp2_tab stays inside
the < 2 ulp bound wherever tests/test_exp2_model.py samples (both sides of the -960 guard included), the bound `k_ld` puts
on the device's Gram entries holds for the model, and the Gram layout the GPU tests compare against."""
import numpy as np
import pytest

import gram_model as gm
import seiso_model as sm
from test_exp2_model import _exp2_tab, _coeffs, _prepare


def _need_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")


def test_vectorised_fma_is_correctly_rounded():
    rng = np.random.default_rng(1)
    n = 20000
    a = rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n))
    b = rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n))
    c = -a * b * (1 + rng.standard_normal(n) * np.exp2(rng.integers(-60, 0, n)))    # heavy cancellation
    c[::3] = rng.standard_normal(n)[::3]
    # ties of the final rounding: c + a b exactly halfway between two doubles
    a[:200], b[:200] = 1.0 + 2.0 ** -30, 1.0 + 2.0 ** -23
    c[:200] = 2.0 ** -53 * np.arange(200)
    got = sm.fma(a, b, c)
    want = np.array([sm.fma_fsum(x, y, z) for x, y, z in zip(a, b, c)])
    assert np.array_equal(got, want)
    plain = a * b + c
    assert np.any(plain != want)                       # the cases do tell a fused from an unfused multiply-add


def test_fma_exp2_tab_within_two_ulp_where_the_no_fma_model_is():
    _need_longdouble()
    co = _coeffs()
    assert sm.coeffs() == co
    rng = np.random.default_rng(3)
    z = -np.concatenate([rng.uniform(0, 1, 20000), rng.uniform(0, 60, 40000), rng.uniform(60, 959.9, 20000),
                         np.arange(0, 961) / 1.0, np.arange(0, 4096) / 64.0, [0.0, 1e-300, 1e-17, 959.999999,
                                                                               959.5, 960.0, 960.0004]])
    for s2 in (1e-15 * 1.0001, 0.37, 1.0, np.exp(0.6), 9.9e14):
        _, tab = _prepare(1.0, s2)
        v = sm.exp2_tab(z, tab)
        want = np.longdouble(s2) * np.exp2(z.astype(np.longdouble))
        rel = np.abs((v.astype(np.longdouble) - want) / want).astype(np.float64)
        assert np.all(np.isfinite(v)) and np.all(v > 0) and rel.max() < 4.5e-16, rel.max()
        v0, _ = _exp2_tab(z, tab, co)
        assert np.all(np.abs(v - v0) <= 2 * np.spacing(v))           # the fma and no-fma models differ in the last bits
        zz = -np.arange(0, 2048) / 64.0                                # exact points: table entry times a power of two
        assert np.array_equal(sm.exp2_tab(zz, tab), np.ldexp(tab[(-np.arange(0, 2048)) & 63], -((np.arange(0, 2048) + 63) // 64)))
        zu = -np.concatenate([[960.0006, 960.0005, 1000.0, 1074.0, 5e4, 1e300], rng.uniform(960.01, 4e6, 2000)])
        assert np.all(sm.exp2_tab(zu, tab) == 0.0)                    # past the guard: a clean zero
    # the guard's granularity: the high word of -960.0004 is that of -960, the one of -960.0006 is not
    assert sm._hi(np.array([-960.0, -960.0004])).tolist() == [sm.GUARD] * 2 and sm._hi(np.array([-960.0006]))[0] > sm.GUARD


def test_device_gram_entries_within_the_k_ld_bound():
    _need_longdouble()
    rng = np.random.default_rng(4)
    for d in (1, 3, 8):
        for ll, ls in ((-6.0, 0.1), (0.0, -0.3), (6.0, 0.5), (0.2, 0.5 * np.log(1.0001e-15)), (0.2, 0.5 * np.log(9.9e14))):
            l2, s2 = np.exp(2 * ll), np.exp(2 * ls)
            sf = sm.prepare(l2, s2)
            X = rng.standard_normal((60, d)) * np.exp(ll) * rng.uniform(0.1, 8, (60, 1))
            X[5] = X[2]
            r2, k, kb = sm.k_ld(X, X, l2, s2)
            dev = sm.exp2_tab(sm.r2_fma(X, X) * sf["c_hi"], sf["tab"])
            err = np.abs((dev - k).astype(np.float64))
            assert np.all(err <= kb), (d, ll, ls, float(np.max(err / kb)))
            assert dev[5, 2] == sf["s2"] and np.all(np.diag(dev) == sf["s2"])     # coincident points: sigma^2 exactly


def test_gram_seiso_layout():
    rng = np.random.default_rng(6)
    N, dx = 130, 4
    Npad, ld = 256, 258
    xp = rng.integers(-64, 65, (N, dx)) / 16.0
    xp[:, 3] = 0.0
    sf = sm.prepare(1.3, 0.7)
    nv = rng.integers(1, 8, N) / 4.0
    G0 = np.full(Npad * ld, -7.0)
    G = sm.gram_seiso(xp.ravel(), dx, N, Npad, sf, nv, N, 0.125, G0, ld).reshape(Npad, ld)
    K = sm.exp2_tab(sm.r2_fma(xp, xp) * sf["c_hi"], sf["tab"])
    assert np.array_equal(G[:N, :N][np.tril_indices(N, -1)], K[np.tril_indices(N, -1)])
    assert np.array_equal(np.diag(G)[:N], np.diag(K) + (nv + 0.125))
    assert np.array_equal(G[:128, :128], G[:128, :128].T)           # the diagonal tile is written whole
    assert np.all(G[:128, 128:] == -7.0) and np.all(G[:, Npad:] == -7.0)    # nothing above the diagonal tiles
    assert np.array_equal(G[N:, N:Npad], np.eye(Npad - N)) and np.all(G[N:Npad, :N] == 0)
    # ownership: the union over the ranks is the single-owner result
    for own_tiles, nranks, axis in ((1, 2, 0), (1, 2, 1), (2, 3, 1)):
        acc = np.array(G0)
        for rank in range(nranks):
            part = sm.gram_seiso(xp.ravel(), dx, N, Npad, sf, nv, N, 0.125, G0, ld, own_tiles, nranks, rank, axis)
            mine = part != G0
            assert not np.any(mine & (acc != G0))
            acc = np.where(mine, part, acc)
        assert np.array_equal(acc, G.ravel())


def test_trace_and_inputs_dx_models_agree_with_a_direct_sum():
    _need_longdouble()
    import gpb200 as g
    rng = np.random.default_rng(7)
    N, d = 150, 3
    X = rng.standard_normal((N, d))
    alpha = rng.standard_normal(N)
    Kinv = rng.standard_normal((N, N))
    l2, s2 = np.exp(2 * 0.3), np.exp(2 * -0.2)
    part, bp, out, bo = sm.trace_seiso(X, N, 256, l2, s2, alpha, Kinv)
    r2, k, _ = sm.k_ld(X, X, l2, s2)
    A = np.outer(alpha, alpha).astype(np.longdouble) - Kinv
    W = np.tril(A, -1) + np.diag(np.diag(A)) / 2
    want = [np.sum(W * k * r2) / np.longdouble(l2), 2 * np.sum(W * k), np.trace(A)]
    assert np.all(np.abs((out - want).astype(float)) <= 1e-15 * np.abs(np.array(want, dtype=float)))
    assert np.all(bo > 0) and np.all(bo < 1e-10 * np.sum(np.abs(part.astype(float)), axis=0))
    for bm_mod, bm_div in ((2, 1), (3, 2)):
        ps = [sm.trace_seiso(X, N, 256, l2, s2, alpha, Kinv, bm_mod, r, bm_div)[0] for r in range(bm_mod)]
        assert np.array_equal(sum(ps), part)
    P = gm.Prog(g.SEIso(0.5 * np.log(l2), 0.5 * np.log(s2)), d)
    o, b = sm.inputs_dx(P, X, alpha, Kinv)
    Asym = np.tril(A) + np.tril(A, -1).T
    dk = -(s2 / l2) * np.exp(-r2 / (2 * np.longdouble(l2)))[:, :, None] * (X[:, None, :] - X[None, :, :])
    want = (Asym[:, :, None] * dk).sum(axis=1)
    assert np.all(np.abs((o - want).astype(float)) <= 1e-14 * np.max(np.abs(want.astype(float))))
    assert np.all(b > 0)
