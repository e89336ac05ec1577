"""numpy model of the dense Gram-family kernels (csrc/gram.cu) and of the kernel-program interpreter they run
(csrc/kprog.cuh).

Pointwise part.  `Prog` holds a flattened program (gpb200.flatten) with its parameters transformed on the host in float64,
as kprog_set_theta does.  `evaluate` restates kprog_eval (every leaf's value and, with grad, its theta-partials kp_leaf<true>
scaled by the adjoint sweep over SUM / PROD) and `evaluate_dx` restates kprog_eval_dx (kp_leaf_dx through the same sweep),
on paired points: row m of A against row m of B.  Every function takes a dtype: np.float64 gives the float64 result,
np.longdouble the extended-precision one.  Each also returns a componentwise bound on |float64 result - exact result|,
derived per leaf from the conditioning of its formula with u = 2^-53 (the constants count the roundings on the path):
  stationary exponentials  k = s exp(-a):    ((n_d + 6) |a| + 4) u |k|           (a = r2 / 2l^2 and its ARD form)
  Matern                   s = sqrt(c) r / l: ((n_d / 2 + 6) s + 10) u |k|
  RQ                       k = s (part)^-alpha, lp = log(part): (alpha (n_d + 6 + 3 |lp|) + 4) u |k|, and the alpha partial
                           k (s / 2part - alpha lp) as a difference of its two terms' bounds (it cancels as s -> 0)
  Periodic                 through delta(sp) = (n_d / 2 + 5) sp u, delta(sin) = |cos| delta(sp) + 2u |sin| and its mirror
                           for cos, so the bound stays meaningful at r near k p (sin -> 0) and k p / 2 (cos -> 0); sin^2
                           to second order, (2 |sin| + delta(sin)) delta(sin), since there delta(sin) may exceed |sin|
  Lin, LinArd, Poly        gamma_{n_d + 1} sum |x_i x_j| through the base; Poly's power by its first-order expansion
  Noise, Const             exact
  SUM / PROD and the adjoint sweep: first-order propagation of the children's bounds, plus u |result| per rounding.
Every component also carries an absolute floor of 64 * 2^-1074 times its scale, for results in or below the subnormal range
(exponent arguments below -708).  No regime is excluded.

Layout part.  Each function reads exactly the elements its kernel reads (an unread element may be NaN) and returns what
the kernel writes (a function that updates a buffer takes it and returns the updated copy; elements the kernel leaves
alone come back unchanged).  Matrices are row-major with an explicit leading dimension, as on the device.  `trace`,
`trace_rect` and `reduce_partials` sum in the kernels' fixed orders: per lane the rows rr = 0..15 of its warp and the
columns b * 64 + 2 lane + e, then the lane tree (shfl_down 16, 8, 4, 2, 1), then the eight warps in order, then per
output the 256-thread strided sums and the shared-memory tree.  On exact operands every order gives the same bits.
"""
import math

import numpy as np

T = 128
LD = np.longdouble
U = 2.0 ** -53
ETA = 2.0 ** -1074
RTOL = 1.4901161193847656e-08               # noise.jl: sqrt(eps(Float64))

SE_ISO, SE_ARD, MAT12_ISO, MAT32_ISO, MAT52_ISO, MAT12_ARD, MAT32_ARD, MAT52_ARD = 1, 2, 3, 4, 5, 6, 7, 8
RQ_ISO, RQ_ARD, PERIODIC, LIN_ISO, LIN_ARD, POLY, NOISE, CONST, SUM, PROD = 9, 10, 11, 12, 13, 14, 15, 16, 32, 33


def gamma(m):
    return m * U / (1 - m * U)


def _m(x):
    return np.abs(np.asarray(x, dtype=np.float64))


def _floor(scale):
    return 64 * ETA * (1.0 + _m(scale))


def set_theta(ops, theta):
    """kprog_set_theta: log-scale theta -> natural-scale parameters, in float64."""
    th = np.asarray(theta, dtype=np.float64)
    par = np.zeros(th.size)
    for op, toff, nth, _, nd, _ in ops:
        t, n = th[toff:toff + nth], nth
        o = par[toff:toff + nth]
        if op == SE_ISO or op in (RQ_ISO, PERIODIC):
            o[0], o[1] = math.exp(2 * t[0]), math.exp(2 * t[1])
            if op != SE_ISO:
                o[2] = math.exp(t[2])
        elif op in (MAT12_ISO, MAT32_ISO, MAT52_ISO, POLY):
            o[0], o[1] = math.exp(t[0]), math.exp(2 * t[1])
        elif op in (SE_ARD, MAT12_ARD, MAT32_ARD, MAT52_ARD):
            o[:n - 1] = [math.exp(-2 * v) for v in t[:n - 1]]
            o[n - 1] = math.exp(2 * t[n - 1])
        elif op == RQ_ARD:
            o[:n - 2] = [math.exp(-2 * v) for v in t[:n - 2]]
            o[n - 2], o[n - 1] = math.exp(2 * t[n - 2]), math.exp(t[n - 1])
        elif op in (LIN_ISO, NOISE, CONST):
            o[0] = math.exp(2 * t[0])
        elif op == LIN_ARD:
            o[:n] = [math.exp(v) for v in t[:n]]
    return par


class Prog:
    """A flattened kernel program (gpb200.flatten) at log-scale theta (default: the kernel's own)."""

    def __init__(self, kernel, d, theta=None):
        import gpb200 as g
        ops, dims, th, _ = g.flatten(kernel, d)
        self.ops = [tuple(int(v) for v in o) for o in ops]
        self.dims = [int(v) for v in dims]
        self.theta = np.asarray(th if theta is None else theta, dtype=np.float64)
        self.n_theta = self.theta.size
        self.par = set_theta(self.ops, self.theta)
        self.d = d
        left, stack = [], []
        for q, o in enumerate(self.ops):
            if o[0] in (SUM, PROD):
                stack.pop()
                left.append(stack.pop())
            else:
                left.append(-1)
            stack.append(q)
        self.left = left

    def fast(self):
        """kprog_fast: one SEIso leaf over every input dimension in order (the dense kernels' specialised formula)."""
        o = self.ops[0]
        return len(self.ops) == 1 and o[0] == SE_ISO and o[4] == self.d and self.dims[o[3]:o[3] + o[4]] == list(range(self.d))


def _sumcols(terms, dt):
    s = np.zeros(terms.shape[0], dtype=dt)
    for k in range(terms.shape[1]):                 # k = 0 .. nd-1, as the device loops
        s = s + terms[:, k]
    return s


def _leaf(P, q, A, B, dt, grad):
    """kp_leaf<grad>: value k, bound bk, theta-partials g[p] and bounds bg[p] (lists of arrays over the pairs)."""
    op, toff, nth, doff, nd, extra = P.ops[q]
    dims = P.dims[doff:doff + nd]
    c = [dt(v) for v in P.par[toff:toff + nth]]
    cm = [abs(float(v)) for v in P.par[toff:toff + nth]]
    Ad, Bd = A[:, dims].astype(dt), B[:, dims].astype(dt)
    df = Ad - Bd
    n = A.shape[0]
    zero = np.zeros(n, dtype=dt)
    g, bg = [], []
    if op in (SE_ISO, SE_ARD):
        w = c[:nd] if op == SE_ARD else [dt(1)] * nd
        r = _sumcols(np.stack([df[:, k] * df[:, k] * w[k] for k in range(nd)], 1), dt) if nd else zero
        s2 = c[1] if op == SE_ISO else c[nth - 1]
        a = (dt(0.5) * r / c[0]) if op == SE_ISO else r / dt(2)
        k = s2 * np.exp(-a)
        ek = ((nd + 6) * _m(a) + 4) * U
        bk = ek * _m(k) + _floor(cm[1] if op == SE_ISO else cm[nth - 1])
        if grad:
            if op == SE_ISO:
                g = [r / c[0] * k, dt(2) * k]
                bg = [(ek + 4 * U) * _m(g[0]) + bk * _m(r / c[0]), 2 * bk]
            else:
                for p in range(nd):
                    gp = df[:, p] * df[:, p] * c[p] * k
                    g.append(gp)
                    bg.append((ek + 4 * U) * _m(gp) + bk * _m(df[:, p] * df[:, p] * c[p]))
                g.append(dt(2) * k)
                bg.append(2 * bk)
    elif op in (MAT12_ISO, MAT32_ISO, MAT52_ISO, MAT12_ARD, MAT32_ARD, MAT52_ARD):
        ard = op >= MAT12_ARD
        w = c[:nd] if ard else [dt(1)] * nd
        r = np.sqrt(_sumcols(np.stack([df[:, k] * df[:, k] * w[k] for k in range(nd)], 1), dt) if nd else zero)
        s2 = c[nth - 1] if ard else c[1]
        sc = cm[nth - 1] if ard else cm[1]
        kind = (op - MAT12_ARD) if ard else (op - MAT12_ISO)          # 0: 1/2, 1: 3/2, 2: 5/2
        s = (r if ard else r / c[0]) * (dt(1) if kind == 0 else np.sqrt(dt(3)) if kind == 1 else np.sqrt(dt(5)))
        e = np.exp(-s)
        k = s2 * e * (1 if kind == 0 else (1 + s) if kind == 1 else (1 + s + s * s / dt(3)))
        ek = ((nd / 2 + 6) * _m(s) + 10) * U
        bk = ek * _m(k) + _floor(sc)
        if grad:
            if not ard:
                g0 = [s * k, s2 * s * s * e, s2 / dt(3) * s * s * (1 + s) * e][kind]
                g0 = np.where(r == 0, dt(0), g0)
                g = [g0, dt(2) * k]
                bg = [(ek + 6 * U) * _m(g0) + _floor(sc) * (1 + _m(s) ** 3), 2 * bk]
            else:
                for p in range(nd):
                    wd = df[:, p] * df[:, p] * c[p]
                    with np.errstate(divide="ignore", invalid="ignore"):
                        v = [wd / r * k, dt(3) * s2 * wd * e, dt(5) / dt(3) * s2 * wd * (1 + s) * e][kind]
                    v = np.where(wd > 0, v, dt(0))
                    g.append(v)
                    bg.append((ek + 8 * U) * _m(v) + _floor(sc) * (1 + _m(wd)) * (1 + _m(s)))
                g.append(dt(2) * k)
                bg.append(2 * bk)
    elif op in (RQ_ISO, RQ_ARD):
        ard = op == RQ_ARD
        w = c[:nd] if ard else [dt(1)] * nd
        r = _sumcols(np.stack([df[:, k] * df[:, k] * w[k] for k in range(nd)], 1), dt) if nd else zero
        s2, al = (c[nth - 2], c[nth - 1]) if ard else (c[1], c[2])
        sc, alm = (cm[nth - 2], cm[nth - 1]) if ard else (cm[1], cm[2])
        s = r if ard else r / c[0]
        part = 1 + s / (dt(2) * al)
        lp = np.log(part)
        if grad:
            pw = np.exp(-al * lp)
        else:
            pw = np.power(part, -al)
        k = s2 * pw
        ek = (alm * (nd + 6 + 3 * _m(lp)) + 4) * U
        bk = ek * _m(k) + _floor(sc)
        if grad:
            pw1 = s2 * (pw / part)
            if ard:
                for p in range(nd):
                    gp = (df[:, p] * df[:, p] * c[p]) * pw1
                    g.append(gp)
                    bg.append((ek + 8 * U) * _m(gp) + _floor(sc) * (1 + _m(df[:, p] * df[:, p] * c[p])))
            else:
                g0 = s2 * s * (pw / part)
                g.append(g0)
                bg.append((ek + 8 * U) * _m(g0) + _floor(sc) * (1 + _m(s)))
            g.append(dt(2) * k)
            bg.append(2 * bk)
            t1, t2 = s / (dt(2) * part), al * lp
            bD = (nd + 8) * U * _m(t1) + alm * (nd + 6 + 3 * _m(lp)) * U + U * _m(t1 - t2)
            ga = k * (t1 - t2)
            g.append(ga)
            bg.append(_m(k) * bD + bk * _m(t1 - t2) + U * _m(ga))
    elif op == PERIODIC:
        r = np.sqrt(_sumcols(df * df, dt)) if nd else zero
        l2, s2, per = c
        pi = dt("3.14159265358979323846264338327950288") if dt is LD else dt(3.141592653589793)
        sp = pi * r / per
        sn, cs = np.sin(sp), np.cos(sp)
        t = dt(2) / l2
        A_ = t * (sn * sn)
        k = s2 * np.exp(-A_)
        dsp = (nd / 2 + 5) * _m(sp) * U
        dsn = _m(cs) * dsp + 2 * U * _m(sn) + ETA
        dcs = _m(sn) * dsp + 2 * U * _m(cs) + ETA
        dA = _m(t) * (2 * _m(sn) + dsn) * dsn + 3 * U * _m(A_)      # sin^2 to second order: dsn may exceed |sin|
        bk = _m(k) * (dA + 3 * U) + _floor(cm[1])
        if grad:
            g0 = dt(2) * k * A_
            Pp = sp * t * (dt(2) * sn * cs)
            dP = _m(t) * 2 * (_m(sn * cs) * dsp + _m(sp) * _m(cs) * dsn + _m(sp) * _m(sn) * dcs) + 5 * U * _m(Pp)
            g2 = k * Pp
            g = [g0, dt(2) * k, g2]
            bg = [2 * (_m(A_) * bk + _m(k) * dA + 2 * U * _m(k * A_)), 2 * bk, _m(k) * dP + bk * _m(Pp) + U * _m(g2)]
    elif op in (LIN_ISO, LIN_ARD, POLY):
        terms = Ad * Bd
        sabs = _m(terms).sum(axis=1) if nd else np.zeros(n)
        if op == LIN_ARD:
            pk = [Ad[:, p] * Bd[:, p] * (dt(1) / (c[p] * c[p])) for p in range(nd)]
            k = _sumcols(np.stack(pk, 1), dt) if nd else zero
            sp = sum((_m(v) for v in pk), np.zeros(n))
            bk = (gamma(nd) + 5 * U) * sp + _floor(0)
            if grad:
                g = [dt(-2) * v for v in pk]
                bg = [10 * U * _m(v) + _floor(0) for v in pk]
        else:
            xy = _sumcols(terms, dt) if nd else zero
            if op == LIN_ISO:
                k = xy / c[0]
                bk = (gamma(nd) * sabs + U * _m(xy)) / cm[0] + 2 * U * _m(k) + _floor(0)
                if grad:
                    g, bg = [dt(-2) * k], [2 * bk]
            else:
                deg = extra
                base = c[0] + xy
                db = gamma(nd + 1) * (cm[0] + sabs)
                pw1 = np.ones(n, dtype=dt)
                for _ in range(deg - 1):
                    pw1 = pw1 * base
                pw = pw1 * base if deg >= 1 else np.ones(n, dtype=dt)
                k = c[1] * pw
                mb = _m(base)
                bk = cm[1] * (deg * mb ** max(deg - 1, 0) * db + 2 * deg * U * mb ** deg) + U * _m(k) + _floor(cm[1])
                if grad:
                    dpw1 = max(deg - 1, 0) * mb ** max(deg - 2, 0) * db + 2 * max(deg - 1, 0) * U * mb ** max(deg - 1, 0)
                    g0 = c[0] * dt(deg) * c[1] * pw1
                    g = [g0, dt(2) * k]
                    bg = [cm[0] * deg * cm[1] * dpw1 + 4 * U * _m(g0) + _floor(cm[1]), 2 * bk]
    elif op == NOISE:
        same = np.ones(n, dtype=bool)
        for p in range(nd):
            a, b = Ad[:, p], Bd[:, p]
            same &= np.abs(a - b) <= dt(RTOL) * np.maximum(np.abs(a), np.abs(b))
        k = np.where(same, c[0], dt(0))
        bk = np.zeros(n)
        if grad:
            g, bg = [dt(2) * k], [np.zeros(n)]
    elif op == CONST:
        k = np.full(n, c[0], dtype=dt)
        bk = np.zeros(n)
        if grad:
            g, bg = [dt(2) * k], [np.zeros(n)]
    else:
        raise ValueError("unknown leaf %d" % op)
    return k, bk, g, bg


def _leaf_dx(P, q, A, B, dt):
    """kp_leaf_dx: dk/dA at the leaf's dims, as an (n, nd) array, with its bound."""
    op, toff, nth, doff, nd, extra = P.ops[q]
    dims = P.dims[doff:doff + nd]
    c = [dt(v) for v in P.par[toff:toff + nth]]
    cm = [abs(float(v)) for v in P.par[toff:toff + nth]]
    Ad, Bd = A[:, dims].astype(dt), B[:, dims].astype(dt)
    df = Ad - Bd
    n = A.shape[0]
    if op in (NOISE, CONST):
        return np.zeros((n, nd), dtype=dt), np.zeros((n, nd))
    ard = op in (SE_ARD, MAT12_ARD, MAT32_ARD, MAT52_ARD, RQ_ARD, LIN_ARD)
    w = [dt(1) / (c[p] * c[p]) for p in range(nd)] if op == LIN_ARD else c[:nd] if ard else [dt(1)] * nd
    r2 = _sumcols(np.stack([df[:, k] * df[:, k] * (w[k] if ard else 1) for k in range(nd)], 1), dt)
    lin = op in (LIN_ISO, LIN_ARD, POLY)
    if op == SE_ISO:
        a = dt(0.5) * r2 / c[0]
        f = -c[1] * np.exp(-a) / c[0]
        ef, fs = ((nd + 6) * _m(a) + 6) * U, cm[1] / cm[0]
    elif op == SE_ARD:
        a = r2 / dt(2)
        f = -c[nth - 1] * np.exp(-a)
        ef, fs = ((nd + 6) * _m(a) + 6) * U, cm[nth - 1]
    elif op in (MAT12_ISO, MAT32_ISO, MAT52_ISO, MAT12_ARD, MAT32_ARD, MAT52_ARD):
        r = np.sqrt(r2)
        kind = (op - MAT12_ARD) if ard else (op - MAT12_ISO)
        l = dt(1) if ard else c[0]
        sv = c[nth - 1] if ard else c[1]
        s = r / l * (dt(1) if kind == 0 else np.sqrt(dt(3)) if kind == 1 else np.sqrt(dt(5)))
        with np.errstate(divide="ignore", invalid="ignore"):
            f = [np.where(r == 0, dt(0), -sv * np.exp(-s) / (l * r)), -3 * sv * np.exp(-s) / (l * l),
                 -dt(5) / dt(3) * sv * (1 + s) * np.exp(-s) / (l * l)][kind]
        ef, fs = ((nd / 2 + 6) * _m(s) + 12) * U, (cm[nth - 1] if ard else cm[1]) / (1 if ard else cm[0] ** 2)
    elif op in (RQ_ISO, RQ_ARD):
        al, sv = (c[nth - 1], c[nth - 2]) if ard else (c[2], c[1])
        alm = cm[nth - 1] if ard else cm[2]
        part = 1 + (r2 / (dt(2) * al) if ard else r2 / (dt(2) * c[2] * c[0]))
        lp = np.log(part)
        f = -sv * np.exp(-(al + 1) * lp) / (dt(1) if ard else c[0])
        ef, fs = ((alm + 1) * (nd + 6 + 3 * _m(lp)) + 6) * U, (cm[nth - 2] if ard else cm[1] / cm[0])
    elif op == PERIODIC:
        r = np.sqrt(r2)
        l2, sv, per = c
        pi = dt("3.14159265358979323846264338327950288") if dt is LD else dt(3.141592653589793)
        sp = pi * r / per
        sn, cs = np.sin(sp), np.cos(sp)
        t = dt(2) / l2
        with np.errstate(divide="ignore", invalid="ignore"):
            S = np.where(r == 0, dt(2) * pi / per, dt(2) * sn * cs / r)
        A_ = t * (sn * sn)
        f = -sv * np.exp(-A_) * t * (pi / per) * S
        dsp = (nd / 2 + 5) * _m(sp) * U
        dsn = _m(cs) * dsp + 2 * U * _m(sn) + ETA
        dcs = _m(sn) * dsp + 2 * U * _m(cs) + ETA
        dA = _m(t) * (2 * _m(sn) + dsn) * dsn + 3 * U * _m(A_)      # sin^2 to second order: dsn may exceed |sin|
        with np.errstate(divide="ignore", invalid="ignore"):
            dS = np.where(r == 0, 4 * U * _m(S), 2 * (_m(cs) * dsn + _m(sn) * dcs) / _m(r) + 4 * U * _m(S))
        base = _m(sv * np.exp(-A_) * t * (pi / per))
        bf = base * dS + _m(f) * (dA + 8 * U)
        v = f[:, None] * df
        return v, bf[:, None] * _m(df) + 2 * U * _m(v) + _floor(cm[1] * _m(t) / cm[2])
    elif op == LIN_ISO:
        f = np.full(n, dt(1) / c[0], dtype=dt)
        ef, fs = U, 0
    elif op == LIN_ARD:
        f = np.ones(n, dtype=dt)
        ef, fs = 0, 0
    elif op == POLY:
        deg = extra
        xy = _sumcols(Ad * Bd, dt)
        base = c[0] + xy
        db = gamma(nd + 1) * (cm[0] + _m(Ad * Bd).sum(axis=1))
        pw1 = np.ones(n, dtype=dt)
        for _ in range(deg - 1):
            pw1 = pw1 * base
        f = c[1] * dt(deg) * pw1 if deg >= 1 else np.zeros(n, dtype=dt)
        m = max(deg - 1, 0)
        dpw1 = m * _m(base) ** max(m - 1, 0) * db + 2 * m * U * _m(base) ** m
        v = f[:, None] * Bd
        bf = cm[1] * deg * dpw1 + 3 * U * _m(f)
        return v, bf[:, None] * _m(Bd) + 2 * U * _m(v) + _floor(cm[1])
    else:
        raise ValueError("unknown leaf %d" % op)
    ww = np.array([_m(x) for x in w]) if nd else np.zeros(0)
    ef = np.broadcast_to(np.asarray(ef, dtype=np.float64), (n,))[:, None]
    if lin:
        v = f[:, None] * np.stack([w[p] * Bd[:, p] for p in range(nd)], 1)
        return v, (ef + 4 * U) * _m(v) + _floor(0)
    v = f[:, None] * np.stack([w[p] * df[:, p] for p in range(nd)], 1)
    return v, (ef + 4 * U) * _m(v) + _floor(fs) * (1 + ww[None, :] * _m(df))


def evaluate(P, A, B, dtype=np.float64, grad=False):
    """kprog_eval<grad> on pairs (A[m], B[m]): k (n,), its bound, and with grad g (n_theta, n) and its bound."""
    A, B = np.atleast_2d(A), np.atleast_2d(B)
    n = A.shape[0]
    nq = len(P.ops)
    val, bval = [None] * nq, [None] * nq
    g = np.zeros((P.n_theta, n), dtype=dtype)
    bg = np.zeros((P.n_theta, n))
    for q, o in enumerate(P.ops):
        if o[0] == SUM:
            l, r = P.left[q], q - 1
            val[q] = val[l] + val[r]
            bval[q] = bval[l] + bval[r] + U * _m(val[q])
        elif o[0] == PROD:
            l, r = P.left[q], q - 1
            val[q] = val[l] * val[r]
            bval[q] = _m(val[r]) * bval[l] + _m(val[l]) * bval[r] + bval[l] * bval[r] + U * _m(val[q])
        else:
            val[q], bval[q], gl, bgl = _leaf(P, q, A, B, dtype, grad)
            for p in range(len(gl)):
                g[o[1] + p], bg[o[1] + p] = gl[p], bgl[p]
    if grad and nq > 1:
        adj, badj = [None] * nq, [None] * nq
        adj[nq - 1], badj[nq - 1] = np.ones(n, dtype=dtype), np.zeros(n)
        for q in range(nq - 1, -1, -1):
            o = P.ops[q]
            if o[0] == SUM:
                adj[P.left[q]], badj[P.left[q]] = adj[q], badj[q]
                adj[q - 1], badj[q - 1] = adj[q], badj[q]
            elif o[0] == PROD:
                l, r = P.left[q], q - 1
                adj[l] = adj[q] * val[r]
                badj[l] = _m(val[r]) * badj[q] + _m(adj[q]) * bval[r] + U * _m(adj[l])
                adj[r] = adj[q] * val[l]
                badj[r] = _m(val[l]) * badj[q] + _m(adj[q]) * bval[l] + U * _m(adj[r])
            else:
                for p in range(o[1], o[1] + o[2]):
                    gp = g[p] * adj[q]
                    bg[p] = _m(adj[q]) * bg[p] + _m(g[p]) * badj[q] + bg[p] * badj[q] + U * _m(gp)
                    g[p] = gp
    return val[nq - 1], bval[nq - 1], g, bg


def evaluate_dx(P, A, B, dtype=np.float64):
    """kprog_eval_dx on pairs: dk(A[m], B[m]) / dA[m] as (n, d), and its bound."""
    A, B = np.atleast_2d(A), np.atleast_2d(B)
    n, d = A.shape
    nq = len(P.ops)
    out = np.zeros((n, d), dtype=dtype)
    bout = np.zeros((n, d))
    absum = np.zeros((n, d))
    nterm = np.zeros(d, dtype=int)
    val, bval, adj, badj = [None] * nq, [None] * nq, [None] * nq, [None] * nq
    if nq > 1:
        for q, o in enumerate(P.ops):
            if o[0] in (SUM, PROD):
                l, r = P.left[q], q - 1
                val[q] = val[l] + val[r] if o[0] == SUM else val[l] * val[r]
                bval[q] = (bval[l] + bval[r] if o[0] == SUM else _m(val[r]) * bval[l] + _m(val[l]) * bval[r]) + U * _m(val[q])
            else:
                val[q], bval[q], _, _ = _leaf(P, q, A, B, dtype, False)
    adj[nq - 1], badj[nq - 1] = np.ones(n, dtype=dtype), np.zeros(n)
    for q in range(nq - 1, -1, -1):
        o = P.ops[q]
        if o[0] == SUM:
            adj[P.left[q]], badj[P.left[q]] = adj[q], badj[q]
            adj[q - 1], badj[q - 1] = adj[q], badj[q]
        elif o[0] == PROD:
            l, r = P.left[q], q - 1
            adj[l] = adj[q] * val[r]
            badj[l] = _m(val[r]) * badj[q] + _m(adj[q]) * bval[r] + U * _m(adj[l])
            adj[r] = adj[q] * val[l]
            badj[r] = _m(val[l]) * badj[q] + _m(adj[q]) * bval[l] + U * _m(adj[r])
        else:
            v, bv = _leaf_dx(P, q, A, B, dtype)
            for p, k in enumerate(P.dims[o[3]:o[3] + o[4]]):
                t = adj[q] * v[:, p]
                out[:, k] = out[:, k] + t
                bout[:, k] += _m(adj[q]) * bv[:, p] + _m(v[:, p]) * badj[q] + U * _m(t)
                absum[:, k] += _m(t)
                nterm[k] += 1
    bout += gamma(np.maximum(nterm - 1, 0))[None, :] * absum
    return out, bout


# ---- layouts ----------------------------------------------------------------------------------------------------------

def _mat(buf, ld, rows):
    return np.asarray(buf)[:rows * ld].reshape(rows, ld)


def gram_lower(kfun, x, ldx, d, N, Npad, noise, n_noise, nugget, G, ldg, own_tiles=0, nranks=1, rank=0, own_axis=0,
               bm_min=0):
    """gram_lower_kernel: lower tiles (bn <= bm, bm >= bm_min, owned) of K + (noise + nugget) I, identity in the padding."""
    out = np.array(G, dtype=np.float64, copy=True)
    M = _mat(out, ldg, Npad) if Npad else None
    X = _mat(x, ldx, N)[:, :d] if N else np.zeros((0, d))
    K = kfun(X, X) if N else np.zeros((0, 0))
    nv = np.full(N, noise[0]) if n_noise == 1 else np.asarray(noise[:N])
    Tn = Npad // T
    for bm in range(Tn):
        for bn in range(bm + 1):
            if bm < bm_min or (own_tiles > 0 and (((bm if own_axis else bn) // own_tiles) % nranks) != rank):
                continue
            blk = np.zeros((T, T))
            i0, j0 = bm * T, bn * T
            ri, rj = np.arange(i0, i0 + T), np.arange(j0, j0 + T)
            vi, vj = ri[ri < N], rj[rj < N]
            blk[:vi.size, :vj.size] = K[np.ix_(vi, vj)]
            for t in range(T):
                gi = i0 + t
                if j0 <= gi < j0 + T:
                    blk[t, gi - j0] = 1.0 if gi >= N else blk[t, gi - j0] + (nv[gi] + nugget)
            M[i0:i0 + T, j0:j0 + T] = blk
    return out


def crossgram(kfun, xs, ldxs, M, Mpad, x, ldx, N, Npad, d, K, ldk):
    """crossgram_kernel: Mpad x Npad of k(xs_m, x_n), zero padding."""
    out = np.array(K, dtype=np.float64, copy=True)
    if Mpad == 0 or Npad == 0:
        return out
    V = _mat(out, ldk, Mpad)
    V[:, :Npad] = 0.0
    if M and N:
        V[:M, :N] = kfun(_mat(xs, ldxs, M)[:, :d], _mat(x, ldx, N)[:, :d])
    return out


def gram_full(kfun, xs, ldxs, M, Mpad, d, K, ldk):
    return crossgram(kfun, xs, ldxs, M, Mpad, xs, ldxs, M, Mpad, d, K, ldk)


def kdiag(kpair, xs, ldxs, d, M):
    """kdiag_kernel: out[m] = k(xs_m, xs_m)."""
    X = _mat(xs, ldxs, M)[:, :d]
    return kpair(X, X)


def gram_grad_full(gfun, x, ldx, d, N, Npad, D, ldd, row0, rows):
    """gram_grad_full_kernel: rows row0 .. row0 + rows of dK/dtheta_j (Npad wide, zero padding), row row0 + r at D[r * ldd]."""
    out = np.array(D, dtype=np.float64, copy=True)
    if rows == 0 or Npad == 0:
        return out
    V = _mat(out, ldd, rows)
    V[:, :Npad] = 0.0
    X = _mat(x, ldx, N)[:, :d]
    r1 = min(row0 + rows, N)
    if r1 > row0:
        V[:r1 - row0, :N] = gfun(X[row0:r1], X)
    return out


def crossgram_grad(gfun, x1, ldx1, N1, N1pad, x2, ldx2, N2, N2pad, d, D, ldd):
    """crossgram_grad_kernel: N1pad x N2pad of dk(x1_m, x2_n)/dtheta_j, zero padding."""
    return crossgram(gfun, x1, ldx1, N1, N1pad, x2, ldx2, N2, N2pad, d, D, ldd)


def kdiag_grad(gpair, x, ldx, d, N, gv, n_theta):
    """kdiag_grad_kernel: out[p * N + i] = g_i dk(x_i, x_i)/dtheta_p."""
    X = _mat(x, ldx, N)[:, :d]
    G = gpair(X, X)                                   # (n_theta, N)
    return (np.asarray(gv[:N])[None, :] * G).reshape(-1)


def mirror_lower_tiles(F, ld, Npad):
    """mirror_lower_tiles_kernel: F[j, i] = F[i, j] for every element of the strict-lower 128-tiles (others unchanged)."""
    out = np.array(F, dtype=np.float64, copy=True)
    if Npad <= T:
        return out
    src = _mat(np.asarray(F, dtype=np.float64), ld, Npad)
    V = _mat(out, ld, Npad)
    for bm in range(Npad // T):
        for bn in range(bm):
            V[bn * T:(bn + 1) * T, bm * T:(bm + 1) * T] = src[bm * T:(bm + 1) * T, bn * T:(bn + 1) * T].T
    return out


def _lane_tree(v):
    v = np.array(v)
    for o in (16, 8, 4, 2, 1):
        v[..., :32 - o] = v[..., :32 - o] + v[..., o:32]
    return v[..., 0]


def _tile_acc(terms, dt):
    """terms[p, 128, 128] (row r, column c of the tile; 0 where skipped) -> the tile's partial per p, in the kernel's order:
    lane l of warp w sums rows w * 16 + rr, then columns b * 64 + 2l + e; lane tree; warps in order."""
    nacc = terms.shape[0]
    acc = np.zeros((nacc, 8, 32), dtype=dt)
    lanes = np.arange(32)
    for rr in range(16):
        rows = np.arange(8) * 16 + rr
        for b in range(2):
            for e in range(2):
                cols = b * 64 + 2 * lanes + e
                acc = acc + terms[:, rows[:, None], cols[None, :]]
    warp = _lane_tree(acc)                             # (nacc, 8)
    v = np.zeros(nacc, dtype=dt)
    for w8 in range(8):
        v = v + warp[:, w8]
    return v


def reduce_partials(part, tiles, nacc, dt=np.float64):
    """reduce_partials_kernel: out[p] = sum over tiles, 256-thread strided sums then the shared-memory tree."""
    part = np.asarray(part, dtype=dt)[:tiles * nacc].reshape(tiles, nacc) if tiles else np.zeros((0, nacc), dt)
    s = np.zeros((256, nacc), dtype=dt)
    for t0 in range(0, tiles, 256):
        blk = part[t0:t0 + 256]
        s[:blk.shape[0]] = s[:blk.shape[0]] + blk
    o = 128
    while o > 0:
        s[:o] = s[:o] + s[o:2 * o]
        o >>= 1
    return s[0]


def trace(gall, x, ldx, d, N, Npad, alpha, Kinv, ldg, bm_mod=1, bm_rem=0, bm_div=1, dt=np.float64):
    """trace_kernel's terms per tile, for `trace_out`.  gall(Xi, Xj) -> (n_theta, ni, nj) theta-partials.  Reads Kinv's
    lower triangle (and, as a pair, element (i, i + 1) of an even row i, which it discards), alpha and x of the N real
    rows.  Tile rows another rank owns (bm / bm_div mod bm_mod != bm_rem) get a zero partial."""
    Tn = Npad // T
    tiles = Tn * (Tn + 1) // 2
    X = _mat(x, ldx, N)[:, :d].astype(dt) if N else np.zeros((0, d), dt)
    Kv = _mat(Kinv, ldg, N) if N else np.zeros((0, 0))
    a = np.asarray(alpha[:N], dtype=dt)
    parts = []
    for lin in range(tiles):
        bm = int((math.sqrt(8.0 * lin + 1.0) - 1.0) * 0.5)
        while bm * (bm + 1) // 2 > lin:
            bm -= 1
        while (bm + 1) * (bm + 2) // 2 <= lin:
            bm += 1
        bn = lin - bm * (bm + 1) // 2
        gx = None
        if bm_mod > 1 and ((bm // max(bm_div, 1)) % bm_mod) != bm_rem:
            parts.append(None)
            continue
        ri = np.arange(bm * T, bm * T + T)
        rj = np.arange(bn * T, bn * T + T)
        live = (ri[:, None] < N) & (rj[None, :] < N) & (rj[None, :] <= ri[:, None])
        vi, vj = ri[ri < N], rj[rj < N]
        A = np.zeros((T, T), dtype=dt)
        if vi.size and vj.size:
            A[:vi.size, :vj.size] = a[vi][:, None] * a[vj][None, :] - Kv[np.ix_(vi, vj)].astype(dt)
            gx = gall(X[vi], X[vj])
        A = np.where(live, A, dt(0))
        w = np.where(ri[:, None] == rj[None, :], dt(0.5) * A, A)
        diagA = np.where(ri[:, None] == rj[None, :], A, dt(0))
        parts.append((w, diagA, gx, vi.size, vj.size))
    return parts, tiles


def trace_out(parts_tiles, n_theta, fast=False, dt=np.float64):
    """Finish `trace`: per-tile partials in the kernel's order, then reduce_partials."""
    parts, tiles = parts_tiles
    nacc = 3 if fast else n_theta + 1
    P = np.zeros((tiles, nacc), dtype=dt)
    for lin, item in enumerate(parts):
        if item is None:
            continue
        w, diagA, gx, ni, nj = item
        terms = np.zeros((nacc, T, T), dtype=dt)
        if gx is not None:
            nb = nacc - 1
            terms[:nb, :ni, :nj] = w[None, :ni, :nj] * gx[:nb]
        terms[nacc - 1] = diagA
        P[lin] = _tile_acc(terms, dt)
    return P.reshape(-1), reduce_partials(P.reshape(-1), tiles, nacc, dt)


def trace_rect(gall, x1, ldx1, N1, x2, ldx2, N2, d, W, ldw, nacc, dt=np.float64):
    """trace_rect_kernel + reduce_partials_kernel: (part, out[nacc]) of sum W[i, m] dk(x1_i, x2_m)/dtheta_p, tile (bm, bn)
    at lin = bm * tn + bn.  Reads W[i, m] for i < N1, m < N2 (and, as a pair, column N2 of every row when N2 is odd)."""
    tm, tn = -(-N1 // T), -(-N2 // T)
    X1 = _mat(x1, ldx1, N1)[:, :d].astype(dt)
    X2 = _mat(x2, ldx2, N2)[:, :d].astype(dt)
    Wm = _mat(W, ldw, N1)[:, :N2].astype(dt)
    P = np.zeros((tm * tn, nacc), dtype=dt)
    for bm in range(tm):
        for bn in range(tn):
            i0, j0 = bm * T, bn * T
            ni, nj = min(T, N1 - i0), min(T, N2 - j0)
            gx = gall(X1[i0:i0 + ni], X2[j0:j0 + nj])[:nacc]
            terms = np.zeros((nacc, T, T), dtype=dt)
            terms[:, :ni, :nj] = Wm[i0:i0 + ni, j0:j0 + nj][None] * gx
            P[bm * tn + bn] = _tile_acc(terms, dt)
    return P.reshape(-1), reduce_partials(P.reshape(-1), tm * tn, nacc, dt)


# ---- edge regimes -------------------------------------------------------------------------------------------------------

def leaves(d, ll=0.1, la=0.2, deg=2):
    """One kernel per leaf kind over d inputs, length-scale log ll, RQ log alpha la, Poly degree deg."""
    import gpb200 as g
    L = [ll] * d
    return [("SEIso", g.SEIso(ll, 0.1)), ("SEArd", g.SEArd(L, 0.1)), ("Mat12Iso", g.Mat12Iso(ll, 0.1)),
            ("Mat32Iso", g.Mat32Iso(ll, 0.1)), ("Mat52Iso", g.Mat52Iso(ll, 0.1)), ("Mat12Ard", g.Mat12Ard(L, 0.1)),
            ("Mat32Ard", g.Mat32Ard(L, 0.1)), ("Mat52Ard", g.Mat52Ard(L, 0.1)), ("RQIso", g.RQIso(ll, 0.1, la)),
            ("RQArd", g.RQArd(L, 0.1, la)), ("Periodic", g.Periodic(ll, 0.1, 0.3)), ("LinIso", g.LinIso(ll)),
            ("LinArd", g.LinArd(L)), ("Poly", g.Poly(0.0, 0.1, deg)), ("Noise", g.Noise(0.1)), ("Const", g.Const(0.1))]


def edge_table(n=64, seed=7):
    """[(regime, kernel name, kernel, d, A, B)]: paired points (A[m], B[m]) in the regimes where the interpreter's formulas
    lose relative accuracy or change branch."""
    import gpb200 as g
    rng = np.random.default_rng(seed)
    d = 3
    out = []
    A = rng.standard_normal((n, d))
    sgn = np.where(rng.standard_normal((n, d)) < 0, -1.0, 1.0)
    for reg, delta in (("coincident", 0.0), ("diff 1e-8", 1e-8), ("diff 1e-150", 1e-150), ("diff 1e-160 (r2 subnormal)", 1e-160),
                       ("diff 1e-200 (r2 = 0)", 1e-200)):
        B = A + delta * sgn if delta else A.copy()
        out += [(reg, nm, k, d, A, B) for nm, k in leaves(d)]
    B = rng.standard_normal((n, d))
    out += [("generic", nm, k, d, A, B) for nm, k in leaves(d)]
    for ll in (-6.0, 6.0):
        out += [("ell = e^%+d" % ll, nm, k, d, A * (math.exp(ll) if ll < 0 else 1.0), B * (math.exp(ll) if ll < 0 else 1.0))
                for nm, k in leaves(d, ll=ll)]
    for la in (-5.0, 5.0):
        out += [("RQ alpha = e^%+d" % la, nm, k, d, A, B) for nm, k in leaves(d, la=la) if nm.startswith("RQ")]
    # exponent arguments across the edge of the normal range (-708) and past total underflow (-745): SE (r^2 / 2) and
    # Matern-1/2 (r) over the same sweep; the other stationary leaves go further
    a = np.linspace(700.0, 760.0, n // 2)
    r = np.concatenate([np.sqrt(2 * a), a])
    u = rng.standard_normal((n, d))
    u /= np.linalg.norm(u, axis=1)[:, None]
    out += [("exp argument 700 .. 760", nm, k, d, A, A + r[:, None] * u) for nm, k in leaves(d, ll=0.0)
            if nm not in ("LinIso", "LinArd", "Poly")]
    # Periodic at r = k p and k p / 2, exactly (as rounded) and off by 1e-12 and 1e-8 relative
    per = math.exp(0.3)
    ks = np.arange(1, 9)
    rr = np.concatenate([ks * per, ks * per / 2])
    rr = np.concatenate([rr, rr * (1 + 1e-12), rr * (1 - 1e-8), rr * (1 + 1e-8)])[:n]
    Bp = A.copy()
    Bp[:, 0] = A[:, 0] + rr
    out += [("Periodic r ~ k p, k p / 2", "Periodic", g.Periodic(0.0, 0.1, 0.3), d, A, Bp)]
    # Poly with a negative base c + x.y (c = 1): x.y around -1, and far below
    t = np.concatenate([-1 + np.linspace(-0.5, 0.5, n // 2), -np.linspace(2, 50, n - n // 2)])
    Ap = np.zeros((n, d))
    Ap[:, 0] = 1.0
    Bq = np.zeros((n, d))
    Bq[:, 0] = t
    Bq[:, 1:] = rng.standard_normal((n, d - 1))
    for deg in (0, 1, 2, 5):
        out.append(("Poly deg %d, negative base" % deg, "Poly", g.Poly(0.0, 0.1, deg), d, Ap, Bq))
    # Noise: |a - b| = rtol max(|a|, |b|) exactly, and one ulp either side
    a0 = 1.5 + np.arange(n // 3) / 64.0
    b0 = a0 - RTOL * a0
    An = np.repeat(A[:n // 3], 1, axis=0).copy()
    An[:, 0] = a0
    rows = []
    for b in (b0, np.nextafter(b0, -np.inf), np.nextafter(b0, np.inf)):
        Bn = An.copy()
        Bn[:, 0] = b
        rows.append((An, Bn))
    out.append(("Noise at the isapprox threshold", "Noise", g.Noise(0.1), d, np.vstack([r_[0] for r_ in rows]),
                np.vstack([r_[1] for r_ in rows])))
    out += [("|x| ~ 1e4", nm, k, d, A * 1e4, B * 1e4) for nm, k in leaves(d) if nm in ("LinIso", "LinArd")]
    # programs: the largest (15 ops: 8 leaves, 7 combinators; a post-order program of binary combinators has an odd
    # length, so GPB200_MAX_OPS = 16 cannot be filled), a product with an exactly zero factor, 96 parameters, Masked
    big = (g.SEIso(0.1, 0.1) + g.RQIso(0.2, 0.1, 0.3)) * (g.Mat32Iso(0.1, 0.0) + g.Periodic(0.0, 0.1, 0.3)) + \
          (g.LinIso(0.5) * g.Const(0.1) + g.Mat52Ard([0.1] * d, 0.2)) * g.Noise(-0.2)
    out.append(("15-op program", "Sum/Prod of 8 leaves", big, d, A, B))
    Az = np.zeros((n, d)); Az[:, 0] = rng.standard_normal(n)
    Bz = np.zeros((n, d)); Bz[:, 1] = rng.standard_normal(n)
    out.append(("product with a zero factor", "SEIso*LinIso", g.SEIso(0.1, 0.2) * g.LinIso(0.3), d, Az, Bz))
    dw = 95
    out.append(("96 parameters", "SEArd(d=95)", g.SEArd(list(np.linspace(-0.5, 0.5, dw)), 0.1), dw,
                rng.standard_normal((n, dw)), rng.standard_normal((n, dw))))
    msk = g.Masked(g.SEIso(0.2, 0.1), [2]) + g.Masked(g.RQArd([0.1, -0.1], 0.1, 0.2), [2, 1]) + \
          g.Masked(g.LinArd([0.3, 0.1]), [1, 1])
    out.append(("Masked, non-leading and repeated dims", "Masked", msk, d, A, B))
    return out


def kmat(P, X1, X2, dtype=np.float64):
    """K(X1, X2) through `evaluate` on every pair."""
    n1, n2 = X1.shape[0], X2.shape[0]
    k = evaluate(P, np.repeat(X1, n2, axis=0), np.tile(X2, (n1, 1)), dtype)[0]
    return k.reshape(n1, n2)


def gmat(P, X1, X2, dtype=np.float64):
    """[dK(X1, X2)/dtheta_p] as (n_theta, n1, n2)."""
    n1, n2 = X1.shape[0], X2.shape[0]
    g = evaluate(P, np.repeat(X1, n2, axis=0), np.tile(X2, (n1, 1)), dtype, grad=True)[2]
    return g.reshape(P.n_theta, n1, n2)
