"""numpy model of the TMA-staged SEIso kernels (csrc/gram_fast.cu: gram_seiso_tma_kernel, trace_seiso_tma_kernel,
reduce_partials3_kernel) and of the training-input gradient (csrc/gram.cu: inputs_dx_kernel).  Builds on tests/gram_model.py.

* `fma` is an exact fused multiply-add in numpy: TwoProduct (Veltkamp/Dekker split) makes a * b = uh + ul exactly, TwoSum makes
  c + uh = th + tl exactly, and RN(th + RO(tl + ul)) with RO = round to odd is the correctly rounded a * b + c (Boldo and
  Melquiond, "Emulation of FMA and correctly rounded sums: proved algorithms using rounding to odd", IEEE TC 2008).
  `fma_fsum` is the scalar restatement with one correctly rounded three-term sum (math.fsum); the CPU tests hold the two
  equal.  With it `exp2_tab` re-executes the kernel's fast exp step by step and gives the device's bits.
* `gram_seiso` restates the TMA Gram's layout bit for bit: r2 by the fma chain over the dx staged columns, exp2_tab(r2 c_hi)
  everywhere, the diagonal's noise + nugget, identity at and past N, whole 128 x 128 lower tiles written (the diagonal tiles'
  upper halves included), nothing above them, tiles another rank owns untouched.  The libm path of a tile with a non-finite
  input is not modelled (the GPU tests hold it by bound and by comparing the other tiles with a clean run).
* `trace_seiso` and `inputs_dx` are long-double references with componentwise bounds that hold whatever the compiler fused.
"""
import math
import os

import numpy as np

import gram_model as gm

T = gm.T
LD = gm.LD
U = gm.U
ETA = gm.ETA
MAGIC = 6755399441055744.0                      # 1.5 * 2^52
LOG2E = "1.442695040888963407359924681001892137"
GUARD = 0xC08E0000                              # high word of -960.0


# ---- exact fma ----------------------------------------------------------------------------------------------------------

def _split(a):
    c = 134217729.0 * a                         # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _round_odd_sum(x, y):
    s, e = two_sum(x, y)
    even = (np.ascontiguousarray(s).view(np.int64) & 1) == 0
    step = np.nextafter(s, np.where(e > 0, np.inf, -np.inf))
    return np.where((e != 0) & even, step, s)


def fma(a, b, c):
    """correctly rounded a * b + c, elementwise (finite operands, no overflow, no underflow of the partial products)"""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, dtype=np.float64) for v in (a, b, c)))
    with np.errstate(invalid="ignore", over="ignore"):       # only past exp2_tab's guard, where the result is discarded
        uh, ul = two_prod(a, b)
        th, tl = two_sum(c, uh)
        return th + _round_odd_sum(tl, ul)


def fma_fsum(a, b, c):
    """scalar fma: TwoProduct, then one correctly rounded three-term sum"""
    p, e = two_prod(np.float64(a), np.float64(b))
    return math.fsum([float(p), float(e), float(c)])


# ---- the fast exp -------------------------------------------------------------------------------------------------------

def coeffs():
    """the degree-5 polynomial of exp2_tab, read from the kernel source"""
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "gaussianprocesses.jl_b200", "csrc",
                            "gram_fast.cu")).read()
    body = src[src.index("double exp2_tab("):]
    body = body[:body.index("return ((unsigned)")]
    return [float(re.search(r"double p = ([0-9.eE+-]+);", body).group(1))] + \
        [float(m) for m in re.findall(r"p = fma\(p, f, ([0-9.eE+-]+)\);", body)]


COEFFS = None


def prepare(l2, s2):
    """seiso_fast_prepare on the host (long double): dict(c_hi, il2, s2, tab)."""
    c = LD(-0.5) / LD(l2) * LD(LOG2E)
    tab = (LD(s2) * np.exp2(np.arange(64, dtype=LD) / LD(64))).astype(np.float64)
    return dict(c_hi=float(c), il2=1.0 / l2, s2=float(s2), tab=tab)


def from_device(v):
    """the 67 doubles (c_hi, il2, s2, tab[64]) the harness returns"""
    v = np.asarray(v, dtype=np.float64)
    return dict(c_hi=float(v[0]), il2=float(v[1]), s2=float(v[2]), tab=v[3:67].copy())


def _hi(x):
    return (np.ascontiguousarray(x, dtype=np.float64).view(np.int64) >> 32) & 0xFFFFFFFF


def exp2_tab(z, tab):
    """exp2_tab(z, tab) of the kernel, bit for bit: s2 2^z for z <= 0, 0 once the high word of z passes that of -960"""
    global COEFFS
    if COEFFS is None:
        COEFFS = coeffs()
    z = np.asarray(z, dtype=np.float64)
    zs = fma(z, 64.0, MAGIC)
    ki = (np.ascontiguousarray(zs).view(np.int64) & 0xFFFFFFFF).astype(np.uint32).view(np.int32).astype(np.int64)
    kf = zs - MAGIC
    f = fma(kf, -0.015625, z)
    p = np.full(z.shape, COEFFS[0])
    for c in COEFFS[1:]:
        p = fma(p, f, c)
    r = np.asarray(tab)[ki & 63] * p
    bits = np.ascontiguousarray(r).view(np.int64)
    hi = (((bits >> 32) + ((ki >> 6) << 20)) & 0xFFFFFFFF)
    v = ((hi << 32) | (bits & 0xFFFFFFFF)).view(np.float64)
    return np.where(_hi(z) > GUARD, 0.0, v)


def r2_fma(Xi, Xj):
    """r2 of every pair (rows of Xi against rows of Xj) by the kernels' chain r2 = fma(df, df, r2) over the staged columns"""
    r2 = np.zeros((Xi.shape[0], Xj.shape[0]))
    for k in range(Xi.shape[1]):
        df = Xi[:, k][:, None] - Xj[:, k][None, :]
        r2 = fma(df, df, r2)
    return r2


# ---- TMA Gram, bit for bit ------------------------------------------------------------------------------------------------

def tri_decode(lin):
    bm = int((math.sqrt(8.0 * lin + 1.0) - 1.0) * 0.5)
    while bm * (bm + 1) // 2 > lin:
        bm -= 1
    while (bm + 1) * (bm + 2) // 2 <= lin:
        bm += 1
    return bm, lin - bm * (bm + 1) // 2


def gram_seiso(xp, dx, N, Npad, sf, noise, n_noise, nugget, G, ldg, own_tiles=0, nranks=1, rank=0, own_axis=0):
    """gram_seiso_tma_kernel on finite inputs: xp holds N rows of dx columns (row pitch dx); G (flat, row pitch ldg) is
    returned updated."""
    out = np.array(G, dtype=np.float64, copy=True)
    M = out[:Npad * ldg].reshape(Npad, ldg)
    X = np.zeros((Npad, dx))
    X[:N] = np.asarray(xp, dtype=np.float64)[:N * dx].reshape(N, dx)        # rows past N: zero-filled by TMA
    nv = np.full(N, noise[0]) if n_noise == 1 else np.asarray(noise[:N], dtype=np.float64)
    Tn = Npad // T
    for bm in range(Tn):
        for bn in range(bm + 1):
            if own_tiles > 0 and (((bm if own_axis else bn) // own_tiles) % nranks) != rank:
                continue
            i0, j0 = bm * T, bn * T
            blk = exp2_tab(r2_fma(X[i0:i0 + T], X[j0:j0 + T]) * sf["c_hi"], sf["tab"])
            gi, gj = np.arange(i0, i0 + T)[:, None], np.arange(j0, j0 + T)[None, :]
            pad = (gi >= N) | (gj >= N)
            on = gi == gj
            blk = np.where(on & ~pad, blk + (nv[np.minimum(gi, N - 1)] + nugget), blk)
            blk = np.where(pad, np.where(on, 1.0, 0.0), blk)
            M[i0:i0 + T, j0:j0 + T] = blk
    return out


# ---- long-double references with bounds -----------------------------------------------------------------------------------

def k_ld(Xi, Xj, l2, s2):
    """(r2, k, bound of the device's k) of SEIso over all pairs: r2 and k in long double.  The device's k carries the
    rounding of r2 (fma chain) and of z = r2 c_hi, |z| ln2 (dx + 2) u relative, and exp2_tab's < 2 ulp plus the rounded
    table and c: ((dx + 4) |a| + 6) u |k| with a = r2 / 2 l2.  Below 2^-960 s2 (|z| > 960) exp2_tab returns 0."""
    d = Xi.shape[1]
    df = Xi.astype(LD)[:, None, :] - Xj.astype(LD)[None, :, :]
    r2 = (df * df).sum(-1)
    a = r2 / (LD(2) * LD(l2))
    k = LD(s2) * np.exp(-a)
    af = a.astype(np.float64)
    b = ((d + 4) * af + 6) * U * k.astype(np.float64) + 64 * ETA * (1 + s2)
    b = b + np.where(af * 1.4426950408889634 > 959.9, s2 * 2.0 ** -959.9, 0.0)
    return r2, k, b


def trace_seiso(X, N, Npad, l2, s2, alpha, Kinv, bm_mod=1, bm_rem=0, bm_div=1):
    """trace_seiso_tma_kernel + reduce_partials3_kernel in long double: per lower tile (lin = bm (bm + 1) / 2 + bn)
      part = { il2 sum w k r2,  2 sum w k,  sum over the diagonal of A },  A = a_i a_j - Kinv_ij over i >= j, i, j < N,
    w = A below the diagonal, A / 2 on it; tiles another rank owns ((bm / bm_div) % bm_mod != bm_rem) give exactly 0.
    Returns (part (tiles, 3), bound of part, out (3), bound of out).  The bounds: every product and the scalings one
    rounding each, r2 gamma_dx, k as `k_ld`, A one rounding (one fma), and gamma_(n + 8) sum |terms| for the sum in any
    order; out adds gamma_(tiles + 9) sum |part| for the reduction."""
    d = X.shape[1]
    Tn = Npad // T
    tiles = Tn * (Tn + 1) // 2
    il2 = LD(1) / LD(l2)
    a = np.asarray(alpha[:N], dtype=LD)
    part = np.zeros((tiles, 3), dtype=LD)
    bnd = np.zeros((tiles, 3))
    for lin in range(tiles):
        bm, bn = tri_decode(lin)
        if bm_mod > 1 and ((bm // bm_div) % bm_mod) != bm_rem:
            continue
        ri = np.arange(bm * T, min(bm * T + T, N))
        rj = np.arange(bn * T, min(bn * T + T, N))
        if ri.size == 0 or rj.size == 0:
            continue
        r2, k, kb = k_ld(X[ri], X[rj], l2, s2)
        A = a[ri][:, None] * a[rj][None, :] - np.asarray(Kinv, dtype=LD)[np.ix_(ri, rj)]
        live = rj[None, :] <= ri[:, None]
        on = rj[None, :] == ri[:, None]
        A = np.where(live, A, LD(0))
        w = np.where(on, A / 2, A)
        t0, t1 = w * k * r2, w * k
        n = int(live.sum())
        g = gm.gamma(n + 8)
        wf, kf, r2f = np.abs(w.astype(np.float64)), k.astype(np.float64), r2.astype(np.float64)
        part[lin] = [il2 * t0.sum(), 2 * t1.sum(), np.where(on, A, LD(0)).sum()]
        bnd[lin, 0] = float(il2) * (g * np.sum(np.abs(t0.astype(np.float64))) + np.sum(wf * r2f * kb) +
                                    (gm.gamma(d) + 4 * U) * np.sum(wf * kf * r2f)) + U * abs(float(part[lin, 0]))
        bnd[lin, 1] = 2 * (g * np.sum(np.abs(t1.astype(np.float64))) + np.sum(wf * kb) + 2 * U * np.sum(wf * kf))
        bnd[lin, 2] = (g + U) * np.sum(np.abs(np.where(on, A, LD(0)).astype(np.float64)))
    out = part.sum(axis=0)
    bout = bnd.sum(axis=0) + gm.gamma(tiles + 9) * np.sum(np.abs(part.astype(np.float64)), axis=0)
    return part, bnd, out, bout


def inputs_dx(P, X, alpha, G, rows=64):
    """inputs_dx_kernel in long double: out[i, :] = sum_j A_ij dk(x_i, x_j)/dx_i over the lower triangle of
    A = alpha alpha' - G (A = -G when alpha is None) mirrored, with the bound
      gamma_(N + 8) sum |A| |d1k| + sum |A| bound(d1k) + sum u (|a_i a_j| + |A|) |d1k|
    (bound(d1k): gm.evaluate_dx; the last term: A formed with or without a fused multiply-add)."""
    N, d = X.shape
    Gl = np.asarray(G, dtype=np.float64)[:N, :N]
    Gs = np.tril(Gl) + np.tril(Gl, -1).T
    aa = np.zeros((N, N)) if alpha is None else np.outer(alpha[:N], alpha[:N])
    A = (aa.astype(LD) if alpha is not None else np.zeros((N, N), LD)) - Gs.astype(LD)
    out = np.zeros((N, d), dtype=LD)
    bnd = np.zeros((N, d))
    for r0 in range(0, N, rows):
        r1 = min(N, r0 + rows)
        nr = r1 - r0
        with np.errstate(all="ignore"):
            v, bv = gm.evaluate_dx(P, np.repeat(X[r0:r1], N, axis=0), np.tile(X, (nr, 1)), LD)
        v, bv = v.reshape(nr, N, d), bv.reshape(nr, N, d)
        Ab = A[r0:r1][:, :, None]
        Af = np.abs(Ab.astype(np.float64))
        vf = np.abs(v.astype(np.float64))
        out[r0:r1] = (Ab * v).sum(axis=1)
        bnd[r0:r1] = gm.gamma(N + 8) * (Af * vf).sum(axis=1) + (Af * bv).sum(axis=1) + \
            U * ((np.abs(aa[r0:r1])[:, :, None] + Af) * vf).sum(axis=1)
    return out, bnd
