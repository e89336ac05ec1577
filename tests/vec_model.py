"""numpy model of the O(N^2) / O(N) kernels that turn the factor into numbers (csrc/vec.cu, csrc/gpa.cu).

Each operation is stated the way the kernels block it and reads exactly what the kernels read:

* blocked triangular solves (trsv_lower_fwd / _bwd and their single-launch forms):
      forward   y_b = W_bb (r_b - sum_{i<b} L_bi y_i),   W_bb = Dinv tile b   (F's diagonal tile is never read)
      backward  a_b = W_bb' (z_b - sum_{i>b} L_ib' a_i), W_bb' = DinvT tile b
  F only needs to support 2-D slicing, so a strided view in which rows overlap works as well as a dense matrix;
* f = L v and u = L' g over the lower triangle of F (gpa_trmv_launch / gpa_trmv_t_launch);
* the GPA scan (gpa_scan_launch): row b of W' is w_c (c >= b; the diagonal tile from DinvT, the rest from G's strict-upper
  tiles), and Z'[b, c] = Z[c, b] = u_c sum_{b<=j<=c} v_j w_j + v_c sum_{j>c} u_j w_j.  Z' goes to F's strict-upper tiles
  beyond the diagonal tile and to ZdT's diagonal tile; ZdT's entries to the left of b are zeroed;
* the fixed-order reductions dot, sum, rowdot, rowvar and rowdot2.

Every function takes a dtype: np.float64 gives the float64 result, np.longdouble the extended-precision one.  The *_bound
functions give componentwise error bounds of the form gamma_k x (the same recurrence on absolute values), derived for any
summation order (so they hold for the kernels' trees, shuffles and carries):

* an inner product of m terms (m - 1 additions after the products, any parenthesisation) satisfies
  |fl(x'y) - x'y| <= gamma_m |x|'|y|, gamma_k = k u / (1 - k u);
* one forward block step, given the computed earlier blocks yhat: the accumulator r_b - sum_{i<b} L_bi yhat_i is an inner
  product of m = 128 b + 1 terms, the product with W_bb one of 128 terms, so
      |yhat_b - W_bb (r_b - sum L_bi yhat_i)| <= (gamma_128 (1 + gamma_m) + gamma_m) |W_bb| (|r_b| + sum |L_bi| |yhat_i|)
                                              <= gamma_{m + 128} |W_bb| (|r_b| + sum |L_bi| |yhat_i|),
  and the same with m = 128 (nb - 1 - b) + 1 backwards;
* f_i = sum_{j<=i} L_ij v_j: gamma_{i+1} (|L||v|)_i;  u_j = sum_{i>=j} L_ij g_i: gamma_{Npad-j} (|L|'|g|)_j;
* the scan: the prefix P_c has c - b + 1 terms and the suffix Q_c has Npad - 1 - c; z = u P + v Q adds one product and one
  addition, so |zhat - z| <= gamma_{len+2} (|u_c| Pabs_c + |v_c| Qabs_c) with len = Npad - b;
* dot / sum / rowdot / rowdot2 of n terms: gamma_n; rowvar: gamma_{N+1} (|kdiag| + sum V^2).

A reference evaluated in long double carries its own error, bounded by the same expression with u = 2^-64; the functions
that return (reference, bound) add it, so |device - reference| <= bound is a complete statement.
"""
import numpy as np

T = 128
U64 = 2.0 ** -53
ULD = float(np.finfo(np.longdouble).eps) / 2
LD = np.longdouble


def gamma(k, u=U64):
    k = np.asarray(k, dtype=np.float64)
    return k * u / (1 - k * u)


def _g2(k):
    """gamma_k for float64 plus gamma_k of the long-double reference, inflated by the rounding of the bound itself"""
    return (gamma(k) + gamma(k, ULD)) * (1 + gamma(k + 4, ULD))


def _c(a, dtype):
    return np.asarray(a, dtype=dtype)


# ---- blocked triangular solves ----------------------------------------------------------------------------------------

def trsv_fwd(F, Dinv, r, dtype=np.float64):
    """y = L^-1 r.  Returns (y, acc); acc_b = r_b - sum_{i<b} L_bi y_i is what the per-step schedule leaves in r."""
    Npad = r.shape[0]
    y = np.zeros(Npad, dtype)
    acc = np.zeros(Npad, dtype)
    for b in range(Npad // T):
        q = b * T
        a = _c(r[q:q + T], dtype)
        if q:
            a = a - _c(F[q:q + T, :q], dtype) @ y[:q]
        acc[q:q + T] = a
        y[q:q + T] = _c(Dinv[q:q + T], dtype) @ a
    return y, acc


def trsv_bwd(F, DinvT, z, dtype=np.float64):
    """a = L^-T z.  Returns (a, acc); acc_b = z_b - sum_{i>b} L_ib' a_i is what the per-step schedule leaves in z."""
    Npad = z.shape[0]
    a = np.zeros(Npad, dtype)
    acc = np.zeros(Npad, dtype)
    for b in reversed(range(Npad // T)):
        q = b * T
        s = _c(z[q:q + T], dtype)
        if q + T < Npad:
            s = s - _c(F[q + T:Npad, q:q + T], dtype).T @ a[q + T:]
        acc[q:q + T] = s
        a[q:q + T] = _c(DinvT[q:q + T], dtype) @ s
    return a, acc


def trsv_fwd_local(F, Dinv, r, yhat):
    """Per block b, with the computed earlier blocks yhat: the long-double W_bb (r_b - sum L_bi yhat_i) and its bound."""
    Npad = r.shape[0]
    ref, bnd = np.zeros(Npad, LD), np.zeros(Npad)
    yl = _c(yhat, LD)
    for b in range(Npad // T):
        q = b * T
        Fb = _c(F[q:q + T, :q], LD)
        a = _c(r[q:q + T], LD) - (Fb @ yl[:q] if q else 0)
        aa = np.abs(_c(r[q:q + T], LD)) + (np.abs(Fb) @ np.abs(yl[:q]) if q else 0)
        W = _c(Dinv[q:q + T], LD)
        ref[q:q + T] = W @ a
        bnd[q:q + T] = _g2(T * (b + 1) + 1) * np.asarray(np.abs(W) @ aa, np.float64)
    return ref, bnd


def trsv_bwd_local(F, DinvT, z, ahat):
    Npad = z.shape[0]
    nb = Npad // T
    ref, bnd = np.zeros(Npad, LD), np.zeros(Npad)
    al = _c(ahat, LD)
    for b in range(nb):
        q = b * T
        s, sa = _c(z[q:q + T], LD), np.abs(_c(z[q:q + T], LD))
        if q + T < Npad:
            Fb = _c(F[q + T:Npad, q:q + T], LD)
            s = s - Fb.T @ al[q + T:]
            sa = sa + np.abs(Fb).T @ np.abs(al[q + T:])
        W = _c(DinvT[q:q + T], LD)
        ref[q:q + T] = W @ s
        bnd[q:q + T] = _g2(T * (nb - b) + 1) * np.asarray(np.abs(W) @ sa, np.float64)
    return ref, bnd


def lower_product(F, Ldiag, y, dtype=np.float64):
    """r = L y for the L whose strictly lower tiles are F's and whose diagonal tiles are Ldiag (Npad x 128, tile b in rows
    b*128 ...): the right-hand side for which the forward recurrence returns y (when Dinv tile b = Ldiag tile b ^-1)."""
    Npad = y.shape[0]
    r = np.zeros(Npad, dtype)
    for b in range(Npad // T):
        q = b * T
        r[q:q + T] = _c(Ldiag[q:q + T], dtype) @ _c(y[q:q + T], dtype)
        if q:
            r[q:q + T] += _c(F[q:q + T, :q], dtype) @ _c(y[:q], dtype)
    return r


def lower_t_product(F, Ldiag, a, dtype=np.float64):
    """z = L' a for the same L (the right-hand side for which the backward recurrence returns a)."""
    Npad = a.shape[0]
    z = np.zeros(Npad, dtype)
    for b in range(Npad // T):
        q = b * T
        z[q:q + T] = _c(Ldiag[q:q + T], dtype).T @ _c(a[q:q + T], dtype)
        if q + T < Npad:
            z[q:q + T] += _c(F[q + T:Npad, q:q + T], dtype).T @ _c(a[q + T:], dtype)
    return z


def trsv_read_mask(Npad, ldf):
    """F elements (Npad x ldf) either solve reads: the strictly lower 128 x 128 tiles"""
    tb = np.arange(Npad) // T
    m = np.zeros((Npad, ldf), bool)
    m[:, :Npad] = tb[None, :] < tb[:, None]
    return m


# ---- GPA: triangular matrix-vector products and the scan ---------------------------------------------------------------

def trmv_read_mask(Npad, ldf):
    """F elements both products read: the lower triangle including the diagonal"""
    m = np.zeros((Npad, ldf), bool)
    m[:, :Npad] = np.tri(Npad, dtype=bool)
    return m


def _tril(F, Npad, dtype):
    return np.where(np.tri(Npad, dtype=bool), _c(F[:Npad, :Npad], dtype), 0)


def trmv(F, v, dtype=np.float64):
    """f_i = sum_{j<=i} L_ij v_j"""
    return _tril(F, v.shape[0], dtype) @ _c(v, dtype)


def trmv_t(F, g, dtype=np.float64):
    """u_j = sum_{i>=j} L_ij g_i"""
    return _tril(F, g.shape[0], dtype).T @ _c(g, dtype)


def trmv_bound(F, v):
    n = v.shape[0]
    return _g2(np.arange(1, n + 1)) * np.asarray(np.abs(_tril(F, n, LD)) @ np.abs(_c(v, LD)), np.float64)


def trmv_t_bound(F, g):
    n = g.shape[0]
    return _g2(n - np.arange(n)) * np.asarray(np.abs(_tril(F, n, LD)).T @ np.abs(_c(g, LD)), np.float64)


def scan_masks(Npad, ld):
    """(G elements read = F elements written: row b, columns tb0 + 128 .. Npad;  DinvT elements read: row b, k >= b - tb0).
    ZdT is written in full: zeros left of b, Z' from b on."""
    b = np.arange(Npad)
    tb0 = b & ~(T - 1)
    c = np.arange(ld)
    fw = (c[None, :] >= (tb0 + T)[:, None]) & (c[None, :] < Npad)
    dr = np.arange(T)[None, :] >= (b - tb0)[:, None]
    return fw, dr


def _wrow(G, DinvT, b, dtype):
    Npad = DinvT.shape[0]
    tb0 = b & ~(T - 1)
    return np.concatenate([_c(DinvT[b, b - tb0:], dtype), _c(G[b, tb0 + T:Npad], dtype)])


def gpa_scan(G, DinvT, u, v, dtype=np.float64):
    """Returns (Zf, ZdT): Zf (Npad x Npad) holds Z' in the written region of F (zeros elsewhere), ZdT (Npad x 128) the
    diagonal tiles of Z' with zeros left of b."""
    Npad = u.shape[0]
    Zf = np.zeros((Npad, Npad), dtype)
    ZdT = np.zeros((Npad, T), dtype)
    uu, vv = _c(u, dtype), _c(v, dtype)
    for b in range(Npad):
        tb0 = b & ~(T - 1)
        w = _wrow(G, DinvT, b, dtype)
        ub, vb = uu[b:], vv[b:]
        P = np.cumsum(vb * w)
        Q = np.concatenate([np.cumsum((ub * w)[::-1])[::-1][1:], np.zeros(1, dtype)])
        z = ub * P + vb * Q
        ZdT[b, b - tb0:] = z[:tb0 + T - b]
        Zf[b, tb0 + T:] = z[tb0 + T - b:]
    return Zf, ZdT


def gpa_scan_bound(G, DinvT, u, v):
    """componentwise bound in the layout of gpa_scan"""
    Npad = u.shape[0]
    Zf = np.zeros((Npad, Npad))
    ZdT = np.zeros((Npad, T))
    ua, va = np.abs(_c(u, LD)), np.abs(_c(v, LD))
    for b in range(Npad):
        tb0 = b & ~(T - 1)
        w = np.abs(_wrow(G, DinvT, b, LD))
        ub, vb = ua[b:], va[b:]
        P = np.cumsum(vb * w)
        Q = np.concatenate([np.cumsum((ub * w)[::-1])[::-1][1:], np.zeros(1, LD)])
        z = np.asarray(_g2(Npad - b + 2) * (ub * P + vb * Q), np.float64)
        ZdT[b, b - tb0:] = z[:tb0 + T - b]
        Zf[b, tb0 + T:] = z[tb0 + T - b:]
    return Zf, ZdT


def scan_lower_Z(Zf, ZdT):
    """Z (Npad x Npad, lower part i >= b) from the scan's output regions: Z[i, b] = Z'[b, i]"""
    Npad = ZdT.shape[0]
    Zt = Zf.copy()
    for b in range(Npad):
        tb0 = b & ~(T - 1)
        Zt[b, b:tb0 + T] = ZdT[b, b - tb0:]
    return np.triu(Zt).T


# ---- fixed-order reductions -------------------------------------------------------------------------------------------

def dot(a, b, n, dtype=np.float64):
    return np.sum(_c(a[:n], dtype) * _c(b[:n], dtype), dtype=dtype)


def dot_bound(a, b, n):
    return float(_g2(n) * np.sum(np.abs(_c(a[:n], LD) * _c(b[:n], LD))))


def vsum(a, n, dtype=np.float64):
    return np.sum(_c(a[:n], dtype), dtype=dtype)


def vsum_bound(a, n):
    return float(_g2(n) * np.sum(np.abs(_c(a[:n], LD))))


def rowdot(K, alpha, M, N, dtype=np.float64):
    """mu_m = sum_{n<N} K[m, n] alpha_n"""
    return _c(K[:M, :N], dtype) @ _c(alpha[:N], dtype)


def rowdot_bound(K, alpha, M, N):
    return _g2(N) * np.asarray(np.abs(_c(K[:M, :N], LD)) @ np.abs(_c(alpha[:N], LD)), np.float64)


def rowvar(V, kdiag, M, N, dtype=np.float64):
    """var_m = kdiag_m - sum_{n<N} V[m, n]^2"""
    Vm = _c(V[:M, :N], dtype)
    return _c(kdiag[:M], dtype) - np.sum(Vm * Vm, axis=1, dtype=dtype)


def rowvar_bound(V, kdiag, M, N):
    Vm = _c(V[:M, :N], LD)
    return _g2(N + 1) * np.asarray(np.abs(_c(kdiag[:M], LD)) + np.sum(Vm * Vm, axis=1), np.float64)


def rowdot2(A, B, M, N, dtype=np.float64):
    """q_m = sum_{n<N} A[m, n] B[m, n]"""
    return np.sum(_c(A[:M, :N], dtype) * _c(B[:M, :N], dtype), axis=1, dtype=dtype)


def rowdot2_bound(A, B, M, N):
    return _g2(N) * np.asarray(np.sum(np.abs(_c(A[:M, :N], LD) * _c(B[:M, :N], LD)), axis=1), np.float64)


# ---- exact operands ---------------------------------------------------------------------------------------------------

def dyadic(rng, shape, k=256):
    """entries j / k, |j| <= k: every product with a small integer and every sum of up to 2^30 of them is exact"""
    return rng.integers(-k, k + 1, size=shape).astype(np.float64) / k


def exact_diag_tiles(rng, nb):
    """(Ldiag, W) stacked Npad x 128: Ldiag_b = I + N_b, W_b = I - N_b = Ldiag_b^-1 exactly (N_b only in rows 64.., columns
    ..64, so N_b^2 = 0).  W_b has no symmetry, so a transposed or misplaced diagonal tile changes the result."""
    Ld = np.zeros((nb * T, T))
    W = np.zeros((nb * T, T))
    for b in range(nb):
        Nb = np.zeros((T, T))
        Nb[64:, :64] = dyadic(rng, (64, 64))
        Ld[b * T:(b + 1) * T] = np.eye(T) + Nb
        W[b * T:(b + 1) * T] = np.eye(T) - Nb
    return Ld, W


def transpose_tiles(D):
    """DinvT from Dinv: every 128 x 128 tile transposed"""
    nb = D.shape[0] // T
    return np.ascontiguousarray(D.reshape(nb, T, T).transpose(0, 2, 1).reshape(nb * T, T))
