// kprog.cuh -- the device "kernel program": a flat post-order description of a covariance
// function (leaves + SUM/PROD) evaluated in registers by the Gram, cross-Gram and gradient-trace
// kernels.  No runtime code generation (north-star: no Triton / CUDA.jl codegen): one interpreter,
// plus compile-time specialisation of the single-leaf SEIso case.
//
// Formulas restate /root/reference/src/kernels/*.jl (cited per leaf below).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include "../../include/gpb200.h"

struct KProg {
    int n_ops;
    int n_theta;
    int fast;                        // 1: single SEIso leaf over dims 0..nd-1 (see kprog_fast)
    int pad_;
    int op[GPB200_MAX_OPS];
    int toff[GPB200_MAX_OPS];
    int nth[GPB200_MAX_OPS];
    int doff[GPB200_MAX_OPS];
    int nd[GPB200_MAX_OPS];
    int extra[GPB200_MAX_OPS];
    int left[GPB200_MAX_OPS];        // combinators: index of the left child (right child = q-1)
    int dims[GPB200_MAX_DIMS];
    double par[GPB200_MAX_THETA];    // transformed parameters (host: exp of the log-scale theta)
};

// The specialised SEIso kernels apply when the program is one SEIso leaf over every input dimension in order.  P.fast
// records the first part from the program alone; d is the input dimension of the points the launch reads.
static inline bool kprog_fast(const KProg& P, int d) { return P.fast && P.nd[0] == d; }

// Host-side transform theta (log scale) -> par (natural scale), mirrors the constructors
// (se_iso.jl:10 SEIso(ll,lσ) = (exp(2ll), exp(2lσ)); se_ard.jl:13 iℓ2 = exp(-2ll); mat12_iso.jl:12
//  ℓ = exp(ll); rq_iso.jl:12 α = exp(lα); periodic.jl:12 p = exp(lp); lin_ard.jl:12 ℓ = exp(ll);
//  poly.jl:12 c = exp(lc)).
static inline void kprog_set_theta(KProg& P, const double* theta) {
    for (int q = 0; q < P.n_ops; ++q) {
        const double* t = theta + P.toff[q];
        double* o = P.par + P.toff[q];
        int n = P.nth[q];
        switch (P.op[q]) {
        case GPB200_OP_SE_ISO:   o[0] = exp(2 * t[0]); o[1] = exp(2 * t[1]); break;
        case GPB200_OP_MAT12_ISO: case GPB200_OP_MAT32_ISO: case GPB200_OP_MAT52_ISO:
                                 o[0] = exp(t[0]); o[1] = exp(2 * t[1]); break;
        case GPB200_OP_SE_ARD: case GPB200_OP_MAT12_ARD: case GPB200_OP_MAT32_ARD: case GPB200_OP_MAT52_ARD:
            for (int k = 0; k < n - 1; ++k) o[k] = exp(-2 * t[k]);
            o[n - 1] = exp(2 * t[n - 1]); break;
        case GPB200_OP_RQ_ISO:   o[0] = exp(2 * t[0]); o[1] = exp(2 * t[1]); o[2] = exp(t[2]); break;
        case GPB200_OP_RQ_ARD:
            for (int k = 0; k < n - 2; ++k) o[k] = exp(-2 * t[k]);
            o[n - 2] = exp(2 * t[n - 2]); o[n - 1] = exp(t[n - 1]); break;
        case GPB200_OP_PERIODIC: o[0] = exp(2 * t[0]); o[1] = exp(2 * t[1]); o[2] = exp(t[2]); break;
        case GPB200_OP_LIN_ISO:  o[0] = exp(2 * t[0]); break;
        case GPB200_OP_LIN_ARD:  for (int k = 0; k < n; ++k) o[k] = exp(t[k]); break;
        case GPB200_OP_POLY:     o[0] = exp(t[0]); o[1] = exp(2 * t[1]); break;
        case GPB200_OP_NOISE: case GPB200_OP_CONST: o[0] = exp(2 * t[0]); break;
        default: break;
        }
    }
}

#ifdef __CUDACC__

// squared Euclidean distance over the leaf's active dims, direct differences
// (distance.jl:43-56 _SqEuclidean_ij; summation order k = 1..dim as the reference's loop)
__device__ __forceinline__ double kp_sqdist(const int* dims, int nd, const double* xi, const double* xj) {
    double s = 0.0;
    for (int k = 0; k < nd; ++k) { double df = xi[dims[k]] - xj[dims[k]]; s += df * df; }
    return s;
}
// weighted (distance.jl:73-80): (x-y)^2 * w_k, summed in order
__device__ __forceinline__ double kp_wsqdist(const int* dims, int nd, const double* w, const double* xi, const double* xj) {
    double s = 0.0;
    for (int k = 0; k < nd; ++k) { double df = xi[dims[k]] - xj[dims[k]]; s += df * df * w[k]; }
    return s;
}
__device__ __forceinline__ double kp_dot(const int* dims, int nd, const double* xi, const double* xj) {
    double s = 0.0;
    for (int k = 0; k < nd; ++k) s += xi[dims[k]] * xj[dims[k]];
    return s;
}

// One leaf: value, and (GRAD) the nth unscaled partials into g[0..nth).
template <bool GRAD>
__device__ __noinline__ double kp_leaf(const KProg& P, int q, const double* xi, const double* xj, double* g) {
    const int* dims = P.dims + P.doff[q];
    const int nd = P.nd[q];
    const double* c = P.par + P.toff[q];
    const int nth = P.nth[q];
    double k = 0.0;
    switch (P.op[q]) {
    case GPB200_OP_SE_ISO: {                       // se_iso.jl:39,41
        double r = kp_sqdist(dims, nd, xi, xj);
        k = c[1] * exp(-0.5 * r / c[0]);
        if (GRAD) { g[0] = r / c[0] * k; g[1] = 2.0 * k; }
    } break;
    case GPB200_OP_SE_ARD: {                       // se_ard.jl:43-50
        double r = kp_wsqdist(dims, nd, c, xi, xj);
        k = c[nth - 1] * exp(-r / 2.0);
        if (GRAD) {
            for (int p = 0; p < nd; ++p) { double df = xi[dims[p]] - xj[dims[p]]; g[p] = df * df * c[p] * k; }
            g[nth - 1] = 2.0 * k;
        }
    } break;
    case GPB200_OP_MAT12_ISO: {                    // mat12_iso.jl:41,43 ; mat.jl:24-26
        double r = sqrt(kp_sqdist(dims, nd, xi, xj));
        k = c[1] * exp(-r / c[0]);
        if (GRAD) { g[0] = (r == 0.0) ? 0.0 : r / c[0] * k; g[1] = 2.0 * k; }
    } break;
    case GPB200_OP_MAT32_ISO: {                    // mat32_iso.jl:41-45
        double r = sqrt(kp_sqdist(dims, nd, xi, xj));
        double s = sqrt(3.0) * r / c[0], e = exp(-s);
        k = c[1] * (1.0 + s) * e;
        if (GRAD) { g[0] = (r == 0.0) ? 0.0 : c[1] * s * s * e; g[1] = 2.0 * k; }
    } break;
    case GPB200_OP_MAT52_ISO: {                    // mat52_iso.jl:40-44
        double r = sqrt(kp_sqdist(dims, nd, xi, xj));
        double s = sqrt(5.0) * r / c[0], e = exp(-s);
        k = c[1] * (1.0 + s + s * s / 3.0) * e;
        if (GRAD) { g[0] = (r == 0.0) ? 0.0 : c[1] / 3.0 * s * s * (1.0 + s) * e; g[1] = 2.0 * k; }
    } break;
    case GPB200_OP_MAT12_ARD: case GPB200_OP_MAT32_ARD: case GPB200_OP_MAT52_ARD: {
        // mat12_ard.jl:43-45, mat32_ard.jl:43-46, mat52_ard.jl:43-47 ; zero-guard mat.jl:5-18
        double r = sqrt(kp_wsqdist(dims, nd, c, xi, xj));
        const double s2 = c[nth - 1];
        const int op = P.op[q];
        double s, e;
        if (op == GPB200_OP_MAT12_ARD) { s = r; e = exp(-r); k = s2 * e; }
        else if (op == GPB200_OP_MAT32_ARD) { s = sqrt(3.0) * r; e = exp(-s); k = s2 * (1.0 + s) * e; }
        else { s = sqrt(5.0) * r; e = exp(-s); k = s2 * (1.0 + s + s * s / 3.0) * e; }
        if (GRAD) {
            for (int p = 0; p < nd; ++p) {
                double df = xi[dims[p]] - xj[dims[p]];
                double wd = df * df * c[p];
                double v;
                if (!(wd > 0.0)) v = 0.0;
                else if (op == GPB200_OP_MAT12_ARD) v = wd / r * k;
                else if (op == GPB200_OP_MAT32_ARD) v = 3.0 * s2 * wd * e;
                else v = 5.0 / 3.0 * s2 * wd * (1.0 + s) * e;
                g[p] = v;
            }
            g[nth - 1] = 2.0 * k;
        }
    } break;
    case GPB200_OP_RQ_ISO: {                       // rq_iso.jl:44-52
        double r = kp_sqdist(dims, nd, xi, xj);
        const double l2 = c[0], s2 = c[1], al = c[2];
        if (!GRAD) k = s2 * pow(1.0 + r / (2.0 * al * l2), -al);
        else {
            // one log + one exp instead of three pow + one log: part^-al = exp(-al log part), part^(-al-1) = part^-al / part
            // (the conditioning w.r.t. the rounding of `part` is the same as pow's; agreement with the oracle ~1e-15)
            const double s = r / l2, part = 1.0 + s / (2.0 * al), lp = log(part), pw = exp(-al * lp);
            k = s2 * pw;
            g[0] = s2 * s * (pw / part);
            g[1] = 2.0 * k;
            g[2] = k * (s / (2.0 * part) - al * lp);
        }
    } break;
    case GPB200_OP_RQ_ARD: {                       // rq_ard.jl:47-54
        double r = kp_wsqdist(dims, nd, c, xi, xj);
        const double s2 = c[nth - 2], al = c[nth - 1];
        if (!GRAD) k = s2 * pow(1.0 + 0.5 * r / al, -al);
        else {
            const double part = 1.0 + r / (2.0 * al), lp = log(part), pw = exp(-al * lp), pw1 = s2 * (pw / part);
            k = s2 * pw;
            for (int p = 0; p < nd; ++p) { double df = xi[dims[p]] - xj[dims[p]]; g[p] = (df * df * c[p]) * pw1; }
            g[nth - 2] = 2.0 * k;
            g[nth - 1] = k * (r / (2.0 * part) - al * lp);
        }
    } break;
    case GPB200_OP_PERIODIC: {                     // periodic.jl:45-51
        double r = sqrt(kp_sqdist(dims, nd, xi, xj));
        const double l2 = c[0], s2 = c[1], per = c[2];
        const double pi = 3.141592653589793;
        if (!GRAD) {
            double sn = sin(pi * r / per);
            k = s2 * exp(-2.0 / l2 * (sn * sn));
        } else {
            // one sincos + one exp instead of three sin + three exp: the reference's three exponentials all have the argument
            // -2 sin^2(pi r / p) / l^2, and sin(2 u) = 2 sin u cos u
            const double sp = pi * r / per, t = 2.0 / l2;
            double sn, cs;
            sincos(sp, &sn, &cs);
            const double e = exp(-t * (sn * sn));
            k = s2 * e;
            g[0] = 2.0 * k * (t * (sn * sn));
            g[1] = 2.0 * k;
            g[2] = k * sp * t * (2.0 * sn * cs);
        }
    } break;
    case GPB200_OP_LIN_ISO: {                      // lin_iso.jl:42,71
        k = kp_dot(dims, nd, xi, xj) / c[0];
        if (GRAD) g[0] = -2.0 * k;
    } break;
    case GPB200_OP_LIN_ARD: {                      // lin_ard.jl:69-75,92
        k = 0.0;
        for (int p = 0; p < nd; ++p) {
            double pk = xi[dims[p]] * xj[dims[p]] * (1.0 / (c[p] * c[p]));
            k += pk;
            if (GRAD) g[p] = -2.0 * pk;
        }
    } break;
    case GPB200_OP_POLY: {                         // poly.jl:44,69-70
        double xy = kp_dot(dims, nd, xi, xj);
        const int deg = P.extra[q];
        double base = c[0] + xy, pw1 = 1.0;        // integer power by repeated multiply (Julia ^Int)
        for (int e = 0; e < deg - 1; ++e) pw1 *= base;
        double pw = (deg >= 1) ? pw1 * base : 1.0;
        k = c[1] * pw;
        if (GRAD) { g[0] = c[0] * deg * c[1] * pw1; g[1] = 2.0 * k; }
    } break;
    case GPB200_OP_NOISE: {                        // noise.jl:31-52: isapprox per coordinate
        bool same = true;
        const double rtol = 1.4901161193847656e-08; // sqrt(eps(Float64))
        for (int p = 0; p < nd; ++p) {
            double a = xi[dims[p]], b = xj[dims[p]];
            if (!(fabs(a - b) <= rtol * fmax(fabs(a), fabs(b)))) { same = false; break; }
        }
        k = same ? c[0] : 0.0;
        if (GRAD) g[0] = 2.0 * k;
    } break;
    case GPB200_OP_CONST: {                        // const.jl:41
        k = c[0];
        if (GRAD) g[0] = 2.0 * k;
    } break;
    default: break;
    }
    return k;
}

// Full program.  GRAD: g[0..n_theta) receives dK/dtheta_p (product rule of prod_kernel.jl:54-68,
// concatenation of sum_kernel.jl:43-51) via one reverse sweep over the post-order list.
template <bool GRAD>
__device__ __forceinline__ double kprog_eval(const KProg& P, const double* xi, const double* xj, double* g) {
    if (P.n_ops == 1) return kp_leaf<GRAD>(P, 0, xi, xj, g);
    double val[GPB200_MAX_OPS];
    for (int q = 0; q < P.n_ops; ++q) {
        const int op = P.op[q];
        if (op == GPB200_OP_SUM) val[q] = val[P.left[q]] + val[q - 1];
        else if (op == GPB200_OP_PROD) val[q] = val[P.left[q]] * val[q - 1];
        else val[q] = kp_leaf<GRAD>(P, q, xi, xj, GRAD ? g + P.toff[q] : g);
    }
    if (GRAD) {
        double adj[GPB200_MAX_OPS];
        adj[P.n_ops - 1] = 1.0;
        for (int q = P.n_ops - 1; q >= 0; --q) {
            const int op = P.op[q];
            if (op == GPB200_OP_SUM) { adj[P.left[q]] = adj[q]; adj[q - 1] = adj[q]; }
            else if (op == GPB200_OP_PROD) { adj[P.left[q]] = adj[q] * val[q - 1]; adj[q - 1] = adj[q] * val[P.left[q]]; }
            else { const double a = adj[q]; double* gl = g + P.toff[q]; for (int p = 0; p < P.nth[q]; ++p) gl[p] *= a; }
        }
    }
    return val[P.n_ops - 1];
}

// Input derivative of one leaf: g1[dims[p]] += s1 * dk(xi, xj)/dxi_p and, if g2, g2[dims[p]] += s2 * the same.  Indexing by
// the global input dimension makes a Masked leaf map itself.  At r = 0 the stationary leaves return the limit of the
// derivative (0, from formulas that carry the difference xi - xj as a factor; Periodic through the guarded sin(2u)/r),
// Mat12 returns 0 where its derivative is undefined; Noise and Const are constant in xi.
static __device__ __noinline__ void kp_leaf_dx(const KProg& P, int q, const double* xi, const double* xj, double s1, double* g1,
                                               double s2, double* g2) {
    const int* dims = P.dims + P.doff[q];
    const int nd = P.nd[q];
    const double* c = P.par + P.toff[q];
    const int nth = P.nth[q];
    const int op = P.op[q];
    // dk/dxi_p = f * w_p * (xi_p - xj_p) for the stationary leaves (w_p = 1 for the isotropic ones), xj_p * w_p for Lin / Poly
    double f = 0.0;
    bool ard = false, lin = false;                  // ard: w_p = c[p] (1 / c[p]^2 for LinArd)
    switch (op) {
    case GPB200_OP_SE_ISO:
        f = -c[1] * exp(-0.5 * kp_sqdist(dims, nd, xi, xj) / c[0]) / c[0]; break;
    case GPB200_OP_SE_ARD:
        f = -c[nth - 1] * exp(-kp_wsqdist(dims, nd, c, xi, xj) / 2.0); ard = true; break;
    case GPB200_OP_MAT12_ISO: {
        const double r = sqrt(kp_sqdist(dims, nd, xi, xj));
        f = (r == 0.0) ? 0.0 : -c[1] * exp(-r / c[0]) / (c[0] * r);
    } break;
    case GPB200_OP_MAT32_ISO: {
        const double s = sqrt(3.0) * sqrt(kp_sqdist(dims, nd, xi, xj)) / c[0];
        f = -3.0 * c[1] * exp(-s) / (c[0] * c[0]);
    } break;
    case GPB200_OP_MAT52_ISO: {
        const double s = sqrt(5.0) * sqrt(kp_sqdist(dims, nd, xi, xj)) / c[0];
        f = -5.0 / 3.0 * c[1] * (1.0 + s) * exp(-s) / (c[0] * c[0]);
    } break;
    case GPB200_OP_MAT12_ARD: case GPB200_OP_MAT32_ARD: case GPB200_OP_MAT52_ARD: {
        const double r = sqrt(kp_wsqdist(dims, nd, c, xi, xj)), sv = c[nth - 1];
        if (op == GPB200_OP_MAT12_ARD) f = (r == 0.0) ? 0.0 : -sv * exp(-r) / r;
        else if (op == GPB200_OP_MAT32_ARD) f = -3.0 * sv * exp(-sqrt(3.0) * r);
        else { const double s = sqrt(5.0) * r; f = -5.0 / 3.0 * sv * (1.0 + s) * exp(-s); }
        ard = true;
    } break;
    case GPB200_OP_RQ_ISO: {
        const double part = 1.0 + kp_sqdist(dims, nd, xi, xj) / (2.0 * c[2] * c[0]);
        f = -c[1] * exp(-(c[2] + 1.0) * log(part)) / c[0];
    } break;
    case GPB200_OP_RQ_ARD: {
        const double al = c[nth - 1], part = 1.0 + kp_wsqdist(dims, nd, c, xi, xj) / (2.0 * al);
        f = -c[nth - 2] * exp(-(al + 1.0) * log(part)); ard = true;
    } break;
    case GPB200_OP_PERIODIC: {
        const double r = sqrt(kp_sqdist(dims, nd, xi, xj));
        const double l2 = c[0], sv = c[1], per = c[2], pi = 3.141592653589793, t = 2.0 / l2;
        double sn, cs;
        sincos(pi * r / per, &sn, &cs);
        const double s2r = (r == 0.0) ? 2.0 * pi / per : 2.0 * sn * cs / r;       // sin(2u) / r, u = pi r / per
        f = -sv * exp(-t * (sn * sn)) * t * (pi / per) * s2r;
    } break;
    case GPB200_OP_LIN_ISO: f = 1.0 / c[0]; lin = true; break;
    case GPB200_OP_LIN_ARD: f = 1.0; lin = ard = true; break;
    case GPB200_OP_POLY: {
        const int deg = P.extra[q];
        const double base = c[0] + kp_dot(dims, nd, xi, xj);
        double pw1 = 1.0;
        for (int e = 0; e < deg - 1; ++e) pw1 *= base;
        f = (deg >= 1) ? c[1] * deg * pw1 : 0.0; lin = true;
    } break;
    default: return;                                // Noise, Const
    }
    for (int p = 0; p < nd; ++p) {
        const int k = dims[p];
        const double w = !ard ? 1.0 : (op == GPB200_OP_LIN_ARD) ? 1.0 / (c[p] * c[p]) : c[p];
        const double v = f * w * (lin ? xj[k] : xi[k] - xj[k]);
        g1[k] += s1 * v;
        if (g2) g2[k] += s2 * v;
    }
}

// dk(xi, xj)/dxi of the full program, accumulated as kp_leaf_dx does: one forward sweep for the node values, the adjoint
// sweep of kprog_eval, then every leaf's input derivative scaled by its adjoint.
__device__ __forceinline__ void kprog_eval_dx(const KProg& P, const double* xi, const double* xj, double s1, double* g1,
                                              double s2, double* g2) {
    if (P.n_ops == 1) { kp_leaf_dx(P, 0, xi, xj, s1, g1, s2, g2); return; }
    double val[GPB200_MAX_OPS], adj[GPB200_MAX_OPS];
    for (int q = 0; q < P.n_ops; ++q) {
        const int op = P.op[q];
        if (op == GPB200_OP_SUM) val[q] = val[P.left[q]] + val[q - 1];
        else if (op == GPB200_OP_PROD) val[q] = val[P.left[q]] * val[q - 1];
        else val[q] = kp_leaf<false>(P, q, xi, xj, nullptr);
    }
    adj[P.n_ops - 1] = 1.0;
    for (int q = P.n_ops - 1; q >= 0; --q) {
        const int op = P.op[q];
        if (op == GPB200_OP_SUM) { adj[P.left[q]] = adj[q]; adj[q - 1] = adj[q]; }
        else if (op == GPB200_OP_PROD) { adj[P.left[q]] = adj[q] * val[q - 1]; adj[q - 1] = adj[q] * val[P.left[q]]; }
        else kp_leaf_dx(P, q, xi, xj, s1 * adj[q], g1, s2 * adj[q], g2);
    }
}

#endif  // __CUDACC__
