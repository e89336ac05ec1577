"""GPU: the two training-input contractions of the sparse engines, called directly through the kernel-contract harness
against numpy (xgrad_oracle.cov_dx for the kernel derivatives):

* rows_dx (gpb200_fitc_cv_kernels which 15): out[row(i)] (+)= sum_j W[i, j] d1k(x_i, u_j) + 2 c_i d1k(x_i, x_i) over the
  unmasked rows, at n in {1, 31, 32, 33, 128} (one warp per row, 8 rows per CTA), M in {1, 128, 300}, d = 1 .. 8 on the
  SEIso register path and on the kernel-program path, d = 12 on the program path, with a row mask, a row map, c, and write
  versus accumulate;
* block_dx (gpb200_fsa_kernels which 12): out[row(i)] (+)= sum_l (G[i, l] + G[l, i]) d1k(x_i, x_l) over the real rows of
  blocks of 1, 127, 128, 129 and 300 points, one item per 128-row tile row;
* the argument errors of both, which launch nothing.

Rows a kernel must not write hold a NaN with its own payload that must come back unchanged; padding holds NaN ("never
read").  Sums of products of kernel derivatives are compared within 1e-12 of sum |w| |d1k|, bitwise across repeated
launches."""
import numpy as np
import pytest

import xgrad_oracle as xo

pytestmark = pytest.mark.gpu

POISON = np.array([0x7FF8_DEAD_0000_0005], dtype=np.uint64).view(np.float64)[0]   # "never read, never written"


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def eng():
    import gpb200
    e = gpb200.Engine(0)
    yield e
    e.close()


def _program(e, kernel, d):
    import gpb200 as g
    ops, dims, theta, _ = g.flatten(kernel, d)
    e.set_kernel(ops, dims, theta.size)
    spec = kernel.spec()
    return theta, (spec[1] if spec[0] == "Fixed" else spec)


def _kernel(kind, d):
    import gpb200 as g
    if kind == "fast":
        return g.SEIso(0.2, 0.1)                                     # the register path whenever d <= 8
    return g.SEArd([0.1 * (k % 3) - 0.1 for k in range(d)], 0.1) + g.LinIso(0.3)   # program path, k(x, x) depends on x


def _run(e, fn, name, args, fargs, launches=1):
    n0 = e.launch_count()
    getattr(e, fn)(name, [int(a) for a in args], fargs)
    assert e.launch_count() - n0 == launches, (name, e.launch_count() - n0)


def _close(got, want, bound):
    assert got.shape == want.shape
    assert np.all(np.isfinite(got))
    err = np.abs(got - want)
    assert np.all(err <= 1e-12 * bound + 1e-300), (np.max(err / (bound + 1e-300)), np.argmax(err))


# ---- rows_dx ---------------------------------------------------------------------------------------------------------------

def _rows_case(e, kind, n, M, d, seed, masked=False, mapped=False, with_c=False, accumulate=False):
    rng = np.random.default_rng(seed)
    theta, spec = _program(e, _kernel(kind, d), d)
    ldx, ldu, ldw = d + 1, d + 2, M + 3
    x = np.full((n, ldx), np.nan); x[:, :d] = rng.uniform(-1.5, 1.5, (n, d))
    u = np.full((M, ldu), np.nan); u[:, :d] = rng.uniform(-1.5, 1.5, (M, d))
    if M and n:
        u[0, :d] = x[0, :d]                                           # a training point on an inducing point
    W = np.full((n, ldw), np.nan); W[:, :M] = rng.standard_normal((n, M))
    c = rng.standard_normal(n) if with_c else None
    mask = (rng.random(n) < 0.7).astype(np.float64) if masked else None
    rows = n + 5
    rmap = rng.permutation(rows)[:n].astype(np.int64) if mapped else np.arange(n, dtype=np.int64)
    out0 = np.full((rows, d), POISON)
    if accumulate:
        out0[rmap] = rng.standard_normal((n, d))
    _, D = xo.cov_dx(spec, x[:, :d], u[:, :d]) if M else (None, np.zeros((n, 0, d)))
    want = out0.copy()
    bound = np.zeros((rows, d))
    live = np.ones(n, bool) if mask is None else mask != 0
    t = np.einsum("ij,ijp->ip", W[:, :M], D)
    b = np.einsum("ij,ijp->ip", np.abs(W[:, :M]), np.abs(D))
    if with_c:
        Dii = xo.kdiag_dx(spec, x[:, :d])                             # 2 d1k(x_i, x_i)
        t += c[:, None] * Dii
        b += np.abs(c[:, None] * Dii)
    want[rmap[live]] = (want[rmap[live]] if accumulate else 0.0) + t[live]
    bound[rmap[live]] = b[live] + (np.abs(out0[rmap[live]]) if accumulate else 0.0)
    dx, du, dW, dout = _dev(x), _dev(u), _dev(W), _dev(out0)
    dc = _dev(c) if with_c else None
    dm = _dev(mask) if masked else None
    dmap = _dev(rmap) if mapped else None
    ptr = lambda t_: t_.data_ptr() if t_ is not None else 0
    args = [ptr(dx), ldx, n, ptr(du), ldu, M, d, ptr(dW), ldw, ptr(dc), ptr(dm), ptr(dmap), ptr(dout), int(accumulate)]
    _run(e, "fitc_cv_kernels", "rows_dx", args, theta, launches=1 if n else 0)
    got = _host(dout)
    dead = np.ones(rows, bool); dead[rmap[live]] = False
    np.testing.assert_array_equal(got[dead].view(np.uint64), want[dead].view(np.uint64))   # untouched, payload kept
    _close(got[~dead], want[~dead], bound[~dead])
    if not accumulate:                                                # a second launch writes the same bits
        _run(e, "fitc_cv_kernels", "rows_dx", args, theta)
        np.testing.assert_array_equal(_host(dout).view(np.uint64), got.view(np.uint64))


@pytest.mark.parametrize("kind", ["fast", "program"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 128])
@pytest.mark.parametrize("M", [1, 128, 300])
def test_rows_dx_sizes(eng, kind, n, M):
    _rows_case(eng, kind, n, M, 3, 100 * n + M)


@pytest.mark.parametrize("kind", ["fast", "program"])
@pytest.mark.parametrize("d", list(range(1, 9)) + [12])
def test_rows_dx_dimensions(eng, kind, d):
    _rows_case(eng, kind, 33, 130, d, d, with_c=True)


@pytest.mark.parametrize("kind", ["fast", "program"])
@pytest.mark.parametrize("masked,mapped,with_c,accumulate", [(True, False, False, False), (False, True, False, False),
                                                              (True, True, True, False), (False, False, True, True),
                                                              (True, True, True, True)])
def test_rows_dx_mask_map_c_accumulate(eng, kind, masked, mapped, with_c, accumulate):
    _rows_case(eng, kind, 77, 129, 4, 7, masked, mapped, with_c, accumulate)


# ---- block_dx ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["fast", "program"])
@pytest.mark.parametrize("accumulate", [False, True])
def test_block_dx_blocks_map_accumulate(eng, kind, accumulate):
    d = 3
    rng = np.random.default_rng(11 + accumulate)
    theta, spec = _program(eng, _kernel(kind, d), d)
    sizes = [1, 127, 128, 129, 300]
    Bs = [-(-n // 128) * 128 for n in sizes]
    Np = sum(Bs)
    N = sum(sizes)
    xb = np.full((Np, d), np.nan)
    G = np.concatenate([np.full(B * B, np.nan) for B in Bs])
    rmap = np.full(Np, -1, dtype=np.int64)
    perm = rng.permutation(N)
    out0 = np.full((N + 3, d), POISON)
    if accumulate:
        out0[:N] = rng.standard_normal((N, d))
    want, bound = out0.copy(), np.zeros((N + 3, d))
    items, P, off, k = [], 0, 0, 0
    dG = None
    blocks = []
    for n, B in zip(sizes, Bs):
        xb[P:P + n] = rng.uniform(-1.5, 1.5, (n, d))
        if n > 2:
            xb[P + 2] = xb[P]                                          # a duplicated input in the block
        Gb = np.full((B, B), np.nan); Gb[:n, :n] = rng.standard_normal((n, n))
        G[off:off + B * B] = Gb.ravel()
        rmap[P:P + n] = perm[k:k + n]
        blocks.append((P, n, B, off))
        _, D = xo.cov_dx(spec, xb[P:P + n], xb[P:P + n])
        S = Gb[:n, :n] + Gb[:n, :n].T
        r = rmap[P:P + n]
        want[r] = (want[r] if accumulate else 0.0) + np.einsum("il,ilp->ip", S, D)
        bound[r] = np.einsum("il,ilp->ip", np.abs(S), np.abs(D)) + (np.abs(out0[r]) if accumulate else 0.0)
        P += B; off += B * B; k += n
    dG, dxb, dmap, dout = _dev(G), _dev(xb), _dev(rmap), _dev(out0)
    for P, n, B, off in blocks:
        for t in range(-(-n // 128)):
            items += [dG.data_ptr() + 8 * off, P, B, n, t]
    args = [dxb.data_ptr(), d, dmap.data_ptr(), dout.data_ptr(), int(accumulate)] + items
    _run(eng, "fsa_kernels", "block_dx", args, theta)
    got = _host(dout)
    np.testing.assert_array_equal(got[N:].view(np.uint64), out0[N:].view(np.uint64))
    _close(got[:N], want[:N], bound[:N])
    if not accumulate:
        _run(eng, "fsa_kernels", "block_dx", args, theta)
        np.testing.assert_array_equal(_host(dout).view(np.uint64), got.view(np.uint64))
    # without a map: row0 + i
    out1 = _dev(np.full((Np, d), POISON))
    _run(eng, "fsa_kernels", "block_dx", [dxb.data_ptr(), d, 0, out1.data_ptr(), 0] + items, theta)
    g1 = _host(out1)
    real = rmap >= 0
    w0 = want[rmap[real]] - (out0[rmap[real]] if accumulate else 0.0)
    _close(g1[real], w0, bound[rmap[real]])
    np.testing.assert_array_equal(g1[~real].view(np.uint64), np.full((int((~real).sum()), d), POISON).view(np.uint64))


# ---- argument errors ---------------------------------------------------------------------------------------------------

def test_argument_errors_launch_nothing(eng):
    d, n, M = 2, 4, 3
    theta, _ = _program(eng, _kernel("fast", d), d)
    buf, obuf = _dev(np.zeros(4096)), _dev(np.zeros(4096))
    p, q = buf.data_ptr(), obuf.data_ptr()
    good = [p, d, n, p, d, M, d, p, M, 0, 0, 0, q, 0]
    _run(eng, "fitc_cv_kernels", "rows_dx", good, theta)
    bad = []
    for i, v in ((0, 0), (3, 0), (7, 0), (12, 0), (1, d - 1), (4, d - 1), (8, M - 1), (2, -1), (5, -1), (13, 2), (6, 200)):
        a = list(good); a[i] = v
        bad.append(("fitc_cv_kernels", "rows_dx", a, theta))
    bad.append(("fitc_cv_kernels", "rows_dx", good[:-1], theta))               # argument count
    bad.append(("fitc_cv_kernels", "rows_dx", good, theta[:-1]))               # theta of n_theta entries
    gitem = [p, 0, 128, 5, 0]
    bgood = [p, d, 0, q, 0] + gitem
    _run(eng, "fsa_kernels", "block_dx", bgood, theta)
    for i, v in ((0, 0), (3, 0), (4, 2), (1, 200)):
        a = list(bgood); a[i] = v
        bad.append(("fsa_kernels", "block_dx", a, theta))
    for i, v in ((0, 0), (1, -1), (2, 100), (2, 0), (3, 129), (3, -1), (4, 1), (4, -1)):
        it = list(gitem); it[i] = v
        bad.append(("fsa_kernels", "block_dx", [p, d, 0, q, 0] + it, theta))
    bad.append(("fsa_kernels", "block_dx", bgood[:-1], theta))                  # not whole items
    for fn, name, a, th in bad:
        n0 = eng.launch_count()
        with pytest.raises(ValueError):
            getattr(eng, fn)(name, a, th)
        assert eng.launch_count() == n0, (name, a)
    # empty sizes launch nothing
    _run(eng, "fitc_cv_kernels", "rows_dx", [p, d, 0, p, d, M, d, p, M, 0, 0, 0, q, 0], theta, launches=0)
    _run(eng, "fsa_kernels", "block_dx", [p, d, 0, q, 0], theta, launches=0)
