"""numpy model of the sparse engine's non-GEMM kernels: the FSA block-diagonal kernels (csrc/fsa.cu), the row kernels of
sparse cross-validation (csrc/fitc_cv.cu) and the FITC element kernels that run between the same GEMMs (csrc/vec.cu).

Each function states one kernel as it reads and writes: it reads exactly the elements the kernel reads (so an unread
element may be NaN) and returns what the kernel writes (functions that update a buffer in place take it and return the
updated copy; elements the kernel leaves alone come back unchanged).  Every function takes a dtype: np.float64 gives the
float64 result, np.longdouble the extended-precision one.

The FSA packed layout is restated from gpb200_fitc_set_blocks (csrc/fsa_engine.cu) by `Layout`: block b of n_b points is
padded to B_b = ceil(n_b / 128) * 128 rows and starts at padded row bstart_b; its B_b x B_b matrix is stored row-major
with leading dimension B_b at offset boff_b of the packed array; rblk maps a padded row to its block, mask is 1 on real
rows and 0 on padding, pos maps a training point to its padded row.  The Gram item list holds the lower tiles of every
block (diag set on diagonal tiles), the gradient list `gtiles` every tile of every block; item offsets are into the
packed array (one staging chunk).

Bounds (componentwise, for any summation order, vec_model.gamma): a sum of m products satisfies
|fl(sum) - sum| <= gamma_m sum |products|.  So
  bdmv          gamma_len sum_k |M_rk| |v_k|       (len = the row's number of terms)
  rowdot        gamma_K   sum_k |A_ik| |v_k|
  trace         gamma_m   sum_ij |w_ij| |g_ij|     (m = the number of (i, j) terms over all tiles), for given g
  delta kind 0  gamma_{ncols+1} (|dk| + 2 sum_m |G_im| |C_im|)
The long-double reference adds its own gamma with u = 2^-64 (vec_model._g2).
"""
import math

import numpy as np

import vec_model as vm

T = 128
LD = np.longdouble


def _c(a, dtype):
    return np.asarray(a, dtype=dtype)


# ---- kernel programs whose values and theta-gradients are exact for dyadic inputs ------------------------------------

def kprog(spec, X1, X2, dtype=np.float64, grad=False):
    """K(X1, X2) and, with grad, [dK/dtheta_p] for the leaves LinIso, LinArd, Poly, Const and Sum / Prod of them, as
    csrc/kprog.cuh evaluates them (parameters transformed on the host in float64, as kprog_set_theta does)."""
    name = spec[0]
    if name in ("Sum", "Prod"):
        Kl, gl = kprog(spec[1], X1, X2, dtype, grad)
        Kr, gr = kprog(spec[2], X1, X2, dtype, grad)
        if name == "Sum":
            return Kl + Kr, gl + gr
        return Kl * Kr, [g * Kr for g in gl] + [Kl * g for g in gr]
    th = [float(t) for t in spec[1]]
    X1, X2 = _c(X1, dtype), _c(X2, dtype)
    dot = X1 @ X2.T
    if name == "LinIso":
        K = dot / _c(math.exp(2 * th[0]), dtype)
        return K, ([-2 * K] if grad else [])
    if name == "LinArd":
        parts = [np.outer(X1[:, p], X2[:, p]) * _c(1.0 / (math.exp(th[p]) * math.exp(th[p])), dtype) for p in range(len(th))]
        return sum(parts, np.zeros((X1.shape[0], X2.shape[0]), dtype)), ([-2 * q for q in parts] if grad else [])
    if name == "Poly":
        c, s2, deg = _c(math.exp(th[0]), dtype), _c(math.exp(2 * th[1]), dtype), int(spec[2])
        base = c + dot
        pw1 = np.ones_like(base)
        for _ in range(deg - 1):
            pw1 = pw1 * base
        K = s2 * (pw1 * base)
        return K, ([c * deg * s2 * pw1, 2 * K] if grad else [])
    if name == "Const":
        K = np.full((X1.shape[0], X2.shape[0]), _c(math.exp(2 * th[0]), dtype))
        return K, ([2 * K] if grad else [])
    raise ValueError("kprog: %r is not one of the exact leaves" % name)


# ---- the FSA packed layout ----------------------------------------------------------------------------------------------

class Layout:
    def __init__(self, sizes, idx=None):
        sizes = [int(s) for s in sizes]
        self.N = sum(sizes)
        idx = np.arange(self.N) if idx is None else np.asarray(idx)
        self.sizes = sizes
        self.bsize = [-(-s // T) * T for s in sizes]
        self.bstart = np.concatenate([[0], np.cumsum(self.bsize)[:-1]]).astype(np.int64)
        self.boff = np.concatenate([[0], np.cumsum([B * B for B in self.bsize])[:-1]]).astype(np.int64)
        self.Np = int(sum(self.bsize))
        self.packed = int(sum(B * B for B in self.bsize))
        self.rblk = np.zeros(self.Np, np.int32)
        self.mask = np.zeros(self.Np)
        self.pos = np.zeros(self.N, np.int64)
        p0 = 0
        for b, (n, B) in enumerate(zip(sizes, self.bsize)):
            P = int(self.bstart[b])
            self.rblk[P:P + B] = b
            self.mask[P:P + n] = 1.0
            self.pos[idx[p0:p0 + n]] = P + np.arange(n)
            p0 += n

    def _tile(self, b, i, j):
        return int(self.boff[b]) + i * T * self.bsize[b] + j * T

    def gram_items(self):
        """(offset, ld, row_i, row_j, diag): the lower tiles of every block"""
        return [(self._tile(b, i, j), B, int(self.bstart[b]) + i * T, int(self.bstart[b]) + j * T, int(i == j))
                for b, B in enumerate(self.bsize) for i in range(B // T) for j in range(i + 1)]

    def gtiles(self):
        """(offset, ld, row_i, row_j, 0): every tile of every block"""
        return [(self._tile(b, i, j), B, int(self.bstart[b]) + i * T, int(self.bstart[b]) + j * T, 0)
                for b, B in enumerate(self.bsize) for i in range(B // T) for j in range(B // T)]

    def block(self, packed, b):
        B = self.bsize[b]
        return packed[int(self.boff[b]):int(self.boff[b]) + B * B].reshape(B, B)

    def dense(self, packed, part):
        """the Np x Np block-diagonal matrix of packed: part 'lower' (k <= r), 'upper' (k >= r) or 'full'"""
        import scipy.linalg as sl
        keep = {"lower": np.tril, "upper": np.triu, "full": lambda a: a}[part]
        return sl.block_diag(*[keep(self.block(packed, b)) for b in range(len(self.bsize)) if self.bsize[b]]) \
            if self.Np else np.zeros((0, 0))


# ---- FSA kernels ----------------------------------------------------------------------------------------------------------

def gram(kfun, xb, items, mask, diag_add, dst, dtype=np.float64):
    """fsa_gram: per item, dst tile (i, j) = k(x_{row_i+i}, x_{row_j+j}) (+ diag_add where row_i+i == row_j+j) on real
    rows, 1 / 0 (identity) where either row is padding; diag items write only i >= j.  kfun(X1, X2) -> K."""
    out = _c(dst, dtype).copy()
    for off, ld, ri, rj, diag in items:
        gi, gj = ri + np.arange(T), rj + np.arange(T)
        real = (mask[gi] != 0)[:, None] & (mask[gj] != 0)[None, :]
        same = gi[:, None] == gj[None, :]
        K = _c(kfun(xb[gi], xb[gj]), dtype)
        v = np.where(real, np.where(same, K + _c(diag_add, dtype), K), np.where(same, 1.0, 0.0).astype(dtype))
        w = np.tril(np.ones((T, T), bool)) if diag else np.ones((T, T), bool)
        view = out[off:off + (T - 1) * ld + T]
        for i in range(T):
            view[i * ld:i * ld + T][w[i]] = v[i][w[i]]
    return out


def bdmv(mode, packed, lay, v, dtype=np.float64):
    """fsa_bdmv: y[r] = sum_{k <= rl} M[rl, k] v[P + k] (mode 0), sum_{k >= rl} (mode 1), sum_{k <= rl} M[rl, k]^2 (mode 2)"""
    y = np.zeros(lay.Np, dtype)
    for b, B in enumerate(lay.bsize):
        if not B:
            continue
        P = int(lay.bstart[b])
        M = _c(lay.block(packed, b), dtype)
        for rl in range(B):
            lo, hi = (rl, B) if mode == 1 else (0, rl + 1)
            row = M[rl, lo:hi]
            y[P + rl] = np.sum(row * row) if mode == 2 else row @ _c(v[P + lo:P + hi], dtype)
    return y


def bdmv_bound(mode, packed, lay, v):
    a = bdmv(mode, np.abs(_c(packed, LD)), lay, None if mode == 2 else np.abs(_c(v, LD)), LD)
    ln = np.concatenate([np.arange(B, 0, -1) if mode == 1 else np.arange(1, B + 1) for B in lay.bsize if B] or [np.zeros(0)])
    return np.asarray(vm._g2(ln) * a, np.float64)


def mask(A, nrows, ncols, rowmask, colmask):
    """fsa_mask: A[i, j] = 0 where rowmask[i] == 0 or colmask[j] == 0 (either may be None), i < nrows, j < ncols"""
    out = A.copy()
    z = np.zeros((nrows, ncols), bool)
    if rowmask is not None:
        z |= (rowmask[:nrows] == 0)[:, None]
    if colmask is not None:
        z |= (colmask[:ncols] == 0)[None, :]
    out[:nrows, :ncols][z] = 0.0
    return out


def permute(scatter, src, pos, n, dst):
    out = dst.copy()
    if scatter:
        out[pos[:n]] = src[:n]
    else:
        out[:n] = src[pos[:n]]
    return out


def resid(a, b, m, n, out, dtype=np.float64):
    o = _c(out, dtype).copy()
    o[:n] = _c(m[:n], dtype) * (_c(a[:n], dtype) - _c(b[:n], dtype))
    return o


def outer(items, a, dst, dtype=np.float64):
    """fsa_outer: dst tile += a[row_i + i] a[row_j + j]"""
    out = _c(dst, dtype).copy()
    for off, ld, ri, rj, _ in items:
        add = np.outer(_c(a[ri:ri + T], dtype), _c(a[rj:rj + T], dtype))
        view = out[off:off + (T - 1) * ld + T]
        for i in range(T):
            view[i * ld:i * ld + T] += add[i]
    return out


def _tile_read(dst, off, ld):
    return np.stack([dst[off + i * ld:off + i * ld + T] for i in range(T)])


def trace_terms(gfun, xb, items, mask, dst, dtype=np.float64):
    """per item (weights w masked to real rows, [dk/dtheta_p]); gfun(X1, X2) -> list of gradient matrices"""
    for off, ld, ri, rj, _ in items:
        gi, gj = ri + np.arange(T), rj + np.arange(T)
        real = (mask[gi] != 0)[:, None] & (mask[gj] != 0)[None, :]
        w = np.where(real, _c(_tile_read(dst, off, ld), dtype), 0)      # masked elements are never read
        yield w, [_c(g, dtype) for g in gfun(xb[gi], xb[gj])], real


def trace(gfun, xb, items, mask, dst, n_theta, dtype=np.float64):
    """fsa_trace: out[p] = sum over items of sum_{ij real} w_ij dk(x_{row_i+i}, x_{row_j+j})/dtheta_p"""
    out = np.zeros(n_theta, dtype)
    for w, g, real in trace_terms(gfun, xb, items, mask, dst, dtype):
        out += np.array([np.sum(np.where(real, w * gp, 0)) for gp in g], dtype)
    return out


def trace_bound(gfun, xb, items, mask, dst, n_theta):
    a = trace(lambda X1, X2: [np.abs(g) for g in gfun(X1, X2)], xb, items, mask, np.abs(dst), n_theta, LD)
    return np.asarray(vm._g2(T * T * len(items)) * a, np.float64)


def axpy_t(C, A, nrows, ncols, alpha, dtype=np.float64):
    """fsa_axpy_t: C[i, j] += alpha A[j, i], i < nrows, j < ncols"""
    out = _c(C, dtype).copy()
    out[:nrows, :ncols] += _c(alpha, dtype) * _c(A[:ncols, :nrows], dtype).T
    return out


def crossgram(kfun, xs, xb, items, mask, dst, dtype=np.float64):
    """fsa_crossgram: dst tile (i, j) = k(xs_{row_i+i}, xb_{row_j+j}), 0 where training row row_j+j is padding"""
    out = _c(dst, dtype).copy()
    for off, ld, ri, rj, _ in items:
        gi, gj = ri + np.arange(T), rj + np.arange(T)
        v = np.where((mask[gj] != 0)[None, :], _c(kfun(xs[gi], xb[gj]), dtype), 0)
        view = out[off:off + (T - 1) * ld + T]
        for i in range(T):
            view[i * ld:i * ld + T] = v[i]
    return out


def rowdot(A, v, K, sq, dtype=np.float64):
    """fsa_rowdot on one item: out[i] = sum_{k < K} A[i, k] v[k] (sq 0) or A[i, k]^2 (sq 1), i < 128"""
    Ak = _c(A[:T, :K], dtype)
    return np.sum(Ak * Ak, axis=1) if sq else Ak @ _c(v[:K], dtype)


def rowdot_bound(A, v, K, sq):
    Ak = np.abs(_c(A[:T, :K], LD))
    return np.asarray(vm._g2(K) * (np.sum(Ak * Ak, axis=1) if sq else Ak @ np.abs(_c(v[:K], LD))), np.float64)


def var(q, g2, r2neg, n, out, dtype=np.float64):
    o = _c(out, dtype).copy()
    o[:n] = _c(q[:n], dtype) - _c(g2[:n], dtype) - _c(r2neg[:n], dtype)
    return o


# ---- sparse cross-validation row kernels ------------------------------------------------------------------------------

def delta(kind, dk, G, C, ncols, nrows, rows_pad, alpha, delta0, da0, dtype=np.float64):
    """fitc_cv delta: kind 0 delta_i = dk_i - 2 G[i, :ncols].C[i, :ncols] (dk_i = dk(x_i, x_i)/dtheta_j), kind 1: 0,
    kind 2: 1; for i < nrows delta_i and da_i = delta_i alpha_i are written, for nrows <= i < rows_pad only da_i = 0."""
    d, a = _c(delta0, dtype).copy(), _c(da0, dtype).copy()
    if kind == 0:
        Gm, Cm = _c(G[:nrows, :ncols], dtype), _c(C[:nrows, :ncols], dtype)
        dl = _c(dk[:nrows], dtype) - 2 * np.sum(Gm * Cm, axis=1)
    else:
        dl = np.full(nrows, 0.0 if kind == 1 else 1.0, dtype)
    d[:nrows] = dl
    a[:nrows] = dl * _c(alpha[:nrows], dtype)
    a[nrows:rows_pad] = 0
    return d, a


def delta_bound(dk, G, C, ncols, nrows):
    Gm, Cm = np.abs(_c(G[:nrows, :ncols], LD)), np.abs(_c(C[:nrows, :ncols], LD))
    return np.asarray(vm._g2(ncols + 1) * (np.abs(_c(dk[:nrows], LD)) + 2 * np.sum(Gm * Cm, axis=1)), np.float64)


def rows(G, Ch, K, P, nrows, ncols, lam, dl, alpha, beta, w, dtype=np.float64):
    """fitc_cv rows: (zja, dg) for i < nrows; G None = 0 (beta unread)"""
    c = lambda a: _c(a, dtype)
    Chm, Km, Pm = c(Ch[:nrows, :ncols]), c(K[:nrows, :ncols]), c(P[:nrows, :ncols])
    if G is None:
        gb = gc = np.zeros(nrows, dtype)
    else:
        Gm = c(G[:nrows, :ncols])
        gb, gc = Gm @ c(beta[:ncols]), np.sum(Gm * Chm, axis=1)
    cw, kc, pc = Chm @ c(w[:ncols]), np.sum(Km * Chm, axis=1), np.sum(Pm * Chm, axis=1)
    il, d = 1 / c(lam[:nrows]), c(dl[:nrows])
    zja = d * c(alpha[:nrows]) * il + gb * il + cw
    dg = d * il * il + 2 * gc * il - 2 * d * kc * il * il + pc
    return zja, dg


def invdiag(lam, q, n, out, dtype=np.float64):
    o = _c(out, dtype).copy()
    il = 1 / _c(lam[:n], dtype)
    o[:n] = il - _c(q[:n], dtype) * il * il
    return o


def eblock(E, G, K, nrows, ncols, lam, dl, dtype=np.float64):
    """E[i, m] += G[i, m] / lam_i - delta_i K[i, m] / lam_i^2 (G None = 0)"""
    o = _c(E, dtype).copy()
    il = (1 / _c(lam[:nrows], dtype))[:, None]
    g = 0 if G is None else _c(G[:nrows, :ncols], dtype) * il
    o[:nrows, :ncols] += g - _c(dl[:nrows], dtype)[:, None] * _c(K[:nrows, :ncols], dtype) * il * il
    return o


def qs(H, R, n, Q, dtype=np.float64):
    o = _c(Q, dtype).copy()
    Rm = _c(R[:n, :n], dtype)
    o[:n, :n] = _c(H[:n, :n], dtype) - Rm - Rm.T
    return o


def wvec(a, b, c, n, w, dtype=np.float64):
    o = _c(w, dtype).copy()
    o[:n] = _c(a[:n], dtype) - _c(b[:n], dtype) - _c(c[:n], dtype)
    return o


def gather(idx, x, d, lam, dl, nv, xout, lamout, delout):
    """rows r < nv: xout[r, :d] = x[idx[r], :d], lamout[r] = lam[idx[r]], delout[r] = delta[idx[r]] (dl None: unwritten)"""
    xo, lo = xout.copy(), lamout.copy()
    do = None if delout is None else delout.copy()
    s = idx[:nv]
    xo[:nv, :d] = x[s, :d]
    lo[:nv] = lam[s]
    if dl is not None:
        do[:nv] = dl[s]
    return xo, lo, do


def diag(out, nv, which, lam, dl, dtype=np.float64):
    """out[r, r] += 1/lam_r (which 0) or delta_r / lam_r^2 (which 1), r < nv"""
    o = _c(out, dtype).copy()
    r = np.arange(nv)
    il = 1 / _c(lam[:nv], dtype)
    o[r, r] += il if which == 0 else _c(dl[:nv], dtype) * il * il
    return o


# ---- FITC element kernels (csrc/vec.cu) ------------------------------------------------------------------------------------

def colscale(A, nrows, ncols, v, dtype=np.float64):
    o = _c(A, dtype).copy()
    o[:nrows, :ncols] *= _c(v[:ncols], dtype)[None, :]
    return o


def scale(mode, A, nrows, ncols, v, dtype=np.float64):
    """mode 0: A[r, j] *= 1/sqrt(v[j]); mode 1: A[r, j] *= 1/v[r]"""
    o = _c(A, dtype).copy()
    f = (1 / np.sqrt(_c(v[:ncols], dtype)))[None, :] if mode == 0 else (1 / _c(v[:nrows], dtype))[:, None]
    o[:nrows, :ncols] *= f
    return o


def fitc_g(alpha, lam, q, n, g, dtype=np.float64):
    o = _c(g, dtype).copy()
    a, il = _c(alpha[:n], dtype), 1 / _c(lam[:n], dtype)
    o[:n] = a * a - (il - _c(q[:n], dtype) * il * il)
    return o


def fitc_wfu(P2, P1, nrows, ncols, alpha, lam, g, beta, dtype=np.float64):
    """P2[i, m] <- 2 alpha_i beta_m - (2/lam_i) P2[i, m] - 2 g_i P1[i, m]"""
    o = _c(P2, dtype).copy()
    c = lambda a: _c(a, dtype)
    o[:nrows, :ncols] = (2 * c(alpha[:nrows])[:, None] * c(beta[:ncols])[None, :] - (2 / c(lam[:nrows]))[:, None] * o[:nrows, :ncols]
                         - 2 * c(g[:nrows])[:, None] * c(P1[:nrows, :ncols]))
    return o


def fitc_wuu(T_, Kinv, Sinv, n, beta, Wuu, dtype=np.float64):
    o = _c(Wuu, dtype).copy()
    c = lambda a: _c(a, dtype)
    b = c(beta[:n])
    o[:n, :n] = c(T_[:n, :n]) - b[:, None] * b[None, :] + c(Kinv[:n, :n]) - c(Sinv[:n, :n])
    return o


def symmetrize(A, n):
    o = A.copy()
    iu = np.triu_indices(n, 1)
    o[iu] = A[:n, :n].T[iu]
    return o
