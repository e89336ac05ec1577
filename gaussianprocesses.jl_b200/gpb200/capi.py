"""ctypes binding of libgpb200.so -- the same C ABI (include/gpb200.h) the Julia shim `ccall`s.

No CPU fallback: if the shared library is missing or no CUDA device is present, construction of an
`Engine` raises.  (The library is built in-tree by `__graft_entry__.build()` / `make -C csrc`.)
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libgpb200.so")

OK, EINVAL, ECUDA, ENCCL, ESTATE = 0, -1, -2, -3, -4

# opcodes (include/gpb200.h)
OP = dict(SE_ISO=1, SE_ARD=2, MAT12_ISO=3, MAT32_ISO=4, MAT52_ISO=5, MAT12_ARD=6, MAT32_ARD=7,
          MAT52_ARD=8, RQ_ISO=9, RQ_ARD=10, PERIODIC=11, LIN_ISO=12, LIN_ARD=13, POLY=14, NOISE=15,
          CONST=16, SUM=32, PROD=33)
MAX_OPS, MAX_THETA, MAX_DIMS, OP_STRIDE = 16, 96, 128, 6

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)
_lp = C.POINTER(C.c_int64)
_H = C.c_void_p

_SIGNATURES = {
    "gpb200_create": (C.c_int, [C.POINTER(_H), C.c_int]),
    "gpb200_destroy": (None, [_H]),
    "gpb200_last_error": (C.c_char_p, [_H]),
    "gpb200_version": (C.c_int, []),
    "gpb200_set_data": (C.c_int, [_H, C.c_int64, C.c_int32, _dp, C.c_int64]),
    "gpb200_set_kernel": (C.c_int, [_H, C.c_int32, _ip, C.c_int32, _ip, C.c_int32]),
    "gpb200_factorize": (C.c_int, [_H, _dp, _dp, C.c_int64, C.c_double]),
    "gpb200_logdet": (C.c_int, [_H, _dp]),
    "gpb200_solve": (C.c_int, [_H, _dp, _dp]),
    "gpb200_mll": (C.c_int, [_H, _dp, _dp, _dp]),
    "gpb200_grad_prepare": (C.c_int, [_H]),
    "gpb200_grad_kernel": (C.c_int, [_H, _dp, _dp, _dp]),
    "gpb200_grad_inputs": (C.c_int, [_H, _dp, _dp]),
    "gpb200_predict": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, _dp, _dp, _dp]),
    "gpb200_predict_grad": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, _dp, _dp, _dp, _dp]),
    "gpb200_rand": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, C.c_int64, _dp, C.c_double, _dp, _dp]),
    "gpb200_append": (C.c_int, [_H, C.c_int64, _dp, C.c_int64]),
    "gpb200_unwhiten": (C.c_int, [_H, _dp, _dp]),
    "gpb200_gpa_grad": (C.c_int, [_H, _dp, _dp, _dp, _dp]),
    "gpb200_cv_param": (C.c_int, [_H, C.c_int32, _dp, _dp, _dp]),
    "gpb200_cv_block": (C.c_int, [_H, C.c_int32, C.c_int64, C.POINTER(C.c_int64), _dp]),
    "gpb200_get_gram": (C.c_int, [_H, _dp]),
    "gpb200_get_factor": (C.c_int, [_H, _dp]),
    "gpb200_get_inverse": (C.c_int, [_H, _dp]),
    "gpb200_get_inverse_diag": (C.c_int, [_H, _dp]),
    "gpb200_get_timings": (C.c_int, [_H, _dp, C.c_int32]),
    "gpb200_launch_count": (C.c_int64, [_H]),
    "gpb200_device_bytes": (C.c_int64, []),
    "gpb200_set_option": (C.c_int, [_H, C.c_char_p, C.c_int64]),
    "gpb200_set_stream": (C.c_int, [_H, C.c_void_p]),
    "gpb200_fp64_peak": (C.c_int, [_H, _dp, _dp]),
    "gpb200_dgemm_nt_device": (C.c_int, [_H, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_void_p,
                                         C.c_int64, C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_int64,
                                         C.c_int, C.c_int, _dp]),
    "gpb200_gemm_nt_desc": (C.c_int, [_H, C.c_int, _lp, C.c_int32, C.c_double, C.c_double]),
    "gpb200_fsa_gemm_items": (C.c_int, [_H, _lp, _dp, C.c_int32]),
    "gpb200_potrf_tiles": (C.c_int, [_H, C.c_int, _lp, C.c_int32, _ip]),
    "gpb200_trsv_tiles": (C.c_int, [_H, C.c_int, C.c_int, _lp, C.c_int32, _ip]),
    "gpb200_gpa_kernels": (C.c_int, [_H, C.c_int, _lp, C.c_int32]),
    "gpb200_row_reductions": (C.c_int, [_H, C.c_int, _lp, C.c_int32]),
    "gpb200_fsa_kernels": (C.c_int, [_H, C.c_int, _lp, C.c_int32, _dp, C.c_int32]),
    "gpb200_gram_kernels": (C.c_int, [_H, C.c_int, _lp, C.c_int32, _dp, C.c_int32]),
    "gpb200_vec_kernels": (C.c_int, [_H, C.c_int, _lp, C.c_int32, _dp, C.c_int32]),
    "gpb200_fitc_cv_kernels": (C.c_int, [_H, C.c_int, _lp, C.c_int32, _dp, C.c_int32]),
    "gpb200_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "gpb200_ipc_export": (C.c_int, [_H, C.c_void_p]),
    "gpb200_ipc_import": (C.c_int, [_H, C.c_int, C.c_void_p]),
    "gpb200_fitc_create": (C.c_int, [C.POINTER(_H), C.c_int]),
    "gpb200_fitc_destroy": (None, [_H]),
    "gpb200_fitc_last_error": (C.c_char_p, [_H]),
    "gpb200_fitc_set_data": (C.c_int, [_H, C.c_int64, C.c_int32, _dp, C.c_int64, C.c_int64, _dp, C.c_int64]),
    "gpb200_fitc_set_kernel": (C.c_int, [_H, C.c_int32, _ip, C.c_int32, _ip, C.c_int32]),
    "gpb200_fitc_factorize": (C.c_int, [_H, _dp, C.c_double]),
    "gpb200_fitc_mll": (C.c_int, [_H, _dp, _dp, _dp, _dp]),
    "gpb200_fitc_grad_noise": (C.c_int, [_H, _dp]),
    "gpb200_fitc_grad_kernel": (C.c_int, [_H, _dp]),
    "gpb200_fitc_grad_kernel_inducing": (C.c_int, [_H, _dp, _dp]),
    "gpb200_fitc_set_inducing": (C.c_int, [_H, C.c_int64, _dp, C.c_int64]),
    "gpb200_fitc_grad_kernel_inputs": (C.c_int, [_H, _dp, _dp, _dp]),
    "gpb200_fitc_set_inputs": (C.c_int, [_H, C.c_int64, _dp, C.c_int64]),
    "gpb200_fitc_append": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, _dp, _dp]),
    "gpb200_fitc_predict": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, _dp]),
    "gpb200_fitc_predict_grad": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, _dp, _dp, _dp]),
    "gpb200_fitc_comm_init": (C.c_int, [_H, C.c_int, C.c_int, C.c_char_p]),
    "gpb200_fitc_predict_cov": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _dp, _dp]),
    "gpb200_fitc_set_mode": (C.c_int, [_H, C.c_int]),
    "gpb200_fitc_set_blocks": (C.c_int, [_H, C.c_int64, _lp, _lp]),
    "gpb200_fitc_predict_fsa": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _lp, _dp, _dp, _dp]),
    "gpb200_fitc_predict_fsa_grad": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _lp, _dp, _dp, _dp, _dp]),
    "gpb200_fitc_get_inverse_diag": (C.c_int, [_H, _dp]),
    "gpb200_fitc_cv_param": (C.c_int, [_H, C.c_int32, _dp, _dp, _dp]),
    "gpb200_fitc_cv_block": (C.c_int, [_H, C.c_int32, C.c_int64, C.POINTER(C.c_int64), _dp]),
    "gpb200_fitc_launch_count": (C.c_int64, [_H]),
    "gpb200_fitc_rand": (C.c_int, [_H, C.c_int64, _dp, C.c_int64, _lp, C.c_int64, _dp, C.c_double, _dp, _dp]),
    "gpb200_fitc_get_timings": (C.c_int, [_H, _dp, C.c_int32]),
    "gpb200_comm_init": (C.c_int, [_H, C.c_int, C.c_int, C.c_char_p]),
    "gpb200_group_create": (C.c_int, [C.POINTER(_H), C.c_int]),
    "gpb200_storage_info": (C.c_int, [_H, C.POINTER(C.c_int64), C.c_int32]),
}

_lib = None


def declared_symbols():
    """Every symbol include/gpb200.h declares (used by the CPU-side ABI test)."""
    return sorted(_SIGNATURES)


def load_library():
    """dlopen libgpb200.so (once).  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libgpb200.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C gaussianprocesses.jl_b200/csrc`.  There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class PosDefException(np.linalg.LinAlgError):
    """Mirror of LinearAlgebra.PosDefException(info) thrown by cholesky! (src/GP.jl:110)."""

    def __init__(self, info):
        super().__init__("matrix is not positive definite; Cholesky factorization failed (leading minor %d)" % info)
        self.info = info


def device_bytes():
    """Bytes of device memory the library's buffers hold now, over every engine of the process (diagnostics)."""
    return int(load_library().gpb200_device_bytes())


def _as_dp(a):
    return a.ctypes.data_as(_dp)


class Engine:
    """Owns one gpb200_handle (one GPU).  Thin, 1:1 with the C ABI."""

    def __init__(self, device=0):
        self._lib = load_library()
        self._h = _H()
        rc = self._lib.gpb200_create(C.byref(self._h), int(device))
        if rc != OK:
            msg = self._lib.gpb200_last_error(None)
            raise RuntimeError("gpb200_create failed (%d): %s" % (rc, msg.decode() if msg else "?"))
        self.N = 0
        self.d = 0
        self.n_theta = 0

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.gpb200_destroy(self._h)
            self._h = _H()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc == OK:
            return
        msg = self._lib.gpb200_last_error(self._h)
        msg = msg.decode() if msg else ""
        if rc > 0:
            raise PosDefException(rc)
        if rc in (EINVAL, ESTATE):
            raise ValueError("%s: %s" % (what, msg))       # ArgumentError on the Julia side
        raise RuntimeError("%s failed (%d): %s" % (what, rc, msg))

    # -- data / model ---------------------------------------------------------------------
    def set_data(self, x_pm):
        """x_pm: (N, d) C-contiguous float64 == Julia's d x N column-major matrix."""
        x_pm = np.ascontiguousarray(x_pm, dtype=np.float64)
        N, d = x_pm.shape
        self._check(self._lib.gpb200_set_data(self._h, N, d, _as_dp(x_pm), d), "set_data")
        self.N, self.d = N, d

    def set_kernel(self, ops, dims, n_theta):
        ops = np.ascontiguousarray(ops, dtype=np.int32).reshape(-1, OP_STRIDE)
        dims = np.ascontiguousarray(dims, dtype=np.int32)
        self._check(self._lib.gpb200_set_kernel(self._h, ops.shape[0], ops.ctypes.data_as(_ip), dims.size,
                                                dims.ctypes.data_as(_ip), int(n_theta)), "set_kernel")
        self.n_theta = int(n_theta)

    def set_option(self, key, value):
        self._check(self._lib.gpb200_set_option(self._h, key.encode(), int(value)), "set_option")

    # -- hot path -------------------------------------------------------------------------
    def factorize(self, theta, log_noise, extra_nugget=0.0):
        theta = np.ascontiguousarray(theta, dtype=np.float64)
        ln = np.ascontiguousarray(np.atleast_1d(log_noise), dtype=np.float64)
        self._check(self._lib.gpb200_factorize(self._h, _as_dp(theta), _as_dp(ln), ln.size, float(extra_nugget)),
                    "factorize")

    def logdet(self):
        out = C.c_double()
        self._check(self._lib.gpb200_logdet(self._h, C.byref(out)), "logdet")
        return out.value

    def solve(self, rhs):
        rhs = np.ascontiguousarray(rhs, dtype=np.float64)
        if rhs.shape != (self.N,):
            raise ValueError("solve: rhs must have length N")
        out = np.empty(self.N)
        self._check(self._lib.gpb200_solve(self._h, _as_dp(rhs), _as_dp(out)), "solve")
        return out

    def mll(self, y_minus_mean):
        r = np.ascontiguousarray(y_minus_mean, dtype=np.float64)
        if r.shape != (self.N,):
            raise ValueError("mll: y must have length N")
        alpha = np.empty(self.N)
        out = C.c_double()
        self._check(self._lib.gpb200_mll(self._h, _as_dp(r), _as_dp(alpha), C.byref(out)), "mll")
        return alpha, out.value

    def grad_prepare(self):
        self._check(self._lib.gpb200_grad_prepare(self._h), "grad_prepare")

    def grad_kernel(self, alpha=None):
        g = np.empty(max(self.n_theta, 1))
        tr = C.c_double()
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_grad_kernel(self._h, ap, _as_dp(g), C.byref(tr)), "grad_kernel")
        return g[:self.n_theta].copy(), tr.value

    def grad_inputs(self, alpha=None):
        """(N, d): sum_j A_ij dk(x_i, x_j)/dx_i with A = alpha alpha' - K_y^-1 after grad_prepare, or A = S after gpa_grad
        with the kernel gradient (alpha must then be None); the mean's part is the caller's"""
        out = np.empty((self.N, self.d))
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_grad_inputs(self._h, ap, _as_dp(out)), "grad_inputs")
        return out

    def predict(self, xs_pm, alpha=None, want_var=True, full_cov=False):
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        M, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        mu = np.empty(M)
        var = np.empty(M) if want_var else None
        cov = np.empty((M, M)) if full_cov else None
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_predict(self._h, M, _as_dp(xs_pm), d, ap, _as_dp(mu),
                                             _as_dp(var) if want_var else None,
                                             _as_dp(cov) if full_cov else None), "predict")
        return mu, var, cov

    def predict_grad(self, xs_pm, alpha=None, want_var=True):
        """(mu_minus_mean[M], var[M] or None, dmu (M, d), dvar (M, d) or None): predictions and their gradients with respect to
        the test inputs; var unclamped, the mean function's part left to the caller."""
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        M, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        mu, dmu = np.empty(M), np.empty((M, d))
        var = np.empty(M) if want_var else None
        dvar = np.empty((M, d)) if want_var else None
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_predict_grad(self._h, M, _as_dp(xs_pm), d, ap, _as_dp(mu), _as_dp(var) if want_var else None,
                                                  _as_dp(dmu), _as_dp(dvar) if want_var else None), "predict_grad")
        return mu, var, dmu, dvar

    def rand(self, xs_pm, z, nugget=1e-10, alpha=None):
        """z: (nsamp, M) standard-normal draws (== Julia's M x nsamp column-major).  Returns (mu_minus_mean[M], samples (nsamp, M))."""
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        z = np.ascontiguousarray(z, dtype=np.float64)
        M, d = xs_pm.shape
        if d != self.d or z.ndim != 2 or z.shape[1] != M:
            raise ValueError("rand: inconsistent dimensions")
        mu = np.empty(M)
        out = np.empty_like(z)
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_rand(self._h, M, _as_dp(xs_pm), d, ap, z.shape[0], _as_dp(z), float(nugget), _as_dp(mu),
                                          _as_dp(out)), "rand")
        return mu, out

    def append(self, xnew_pm):
        """extend the factor by the rows of xnew_pm (k, d) with unchanged hyper-parameters (ElasticGPE append!)"""
        xnew_pm = np.ascontiguousarray(xnew_pm, dtype=np.float64)
        k, d = xnew_pm.shape
        if d != self.d:
            raise ValueError("append: wrong input dimension")
        self._check(self._lib.gpb200_append(self._h, k, _as_dp(xnew_pm), d), "append")
        self.N += k

    def unwhiten(self, v):
        """f = L v with L the factor of the last factorize (GPA's latent variables, src/GPA.jl:106,125)."""
        v = np.ascontiguousarray(v, dtype=np.float64)
        if v.shape != (self.N,):
            raise ValueError("unwhiten: v must have length N")
        f = np.empty(self.N)
        self._check(self._lib.gpb200_unwhiten(self._h, _as_dp(v), _as_dp(f)), "unwhiten")
        return f

    def gpa_grad(self, v, dl_df, process=True, kern=True):
        """GPA gradient pieces (src/GPA.jl:164-173, 200): (L' dl_df or None, full kernel-parameter gradient or None).
        The kernel part overwrites K^-1 and the resident alpha on the device."""
        v = np.ascontiguousarray(v, dtype=np.float64)
        g = np.ascontiguousarray(dl_df, dtype=np.float64)
        if v.shape != (self.N,) or g.shape != (self.N,):
            raise ValueError("gpa_grad: v and dl_df must have length N")
        u = np.empty(self.N) if process else None
        gk = np.empty(max(self.n_theta, 1)) if kern else None
        self._check(self._lib.gpb200_gpa_grad(self._h, _as_dp(v), _as_dp(g), _as_dp(u) if process else None,
                                              _as_dp(gk) if kern else None), "gpa_grad")
        return u, (gk[:self.n_theta].copy() if kern else None)

    def cv_param(self, param, alpha=None):
        """(Z_j alpha, diag(Z_j K^-1)) for kernel parameter `param` (index into the full parameter vector) or -1 = noise."""
        za, dg = np.empty(self.N), np.empty(self.N)
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_cv_param(self._h, int(param), ap, _as_dp(za), _as_dp(dg)), "cv_param")
        return za, dg

    def cv_block(self, which, idx):
        idx = np.ascontiguousarray(idx, dtype=np.int64)
        out = np.empty((idx.size, idx.size))
        self._check(self._lib.gpb200_cv_block(self._h, int(which), idx.size, idx.ctypes.data_as(C.POINTER(C.c_int64)), _as_dp(out)), "cv_block")
        return out

    # -- debug ----------------------------------------------------------------------------
    def gram(self):
        K = np.empty((self.N, self.N))
        self._check(self._lib.gpb200_get_gram(self._h, _as_dp(K)), "get_gram")
        return K

    def factor_upper(self):
        """U (upper) with K_y = U'U, as a numpy (N, N) array (row i, col j -> U[i, j])."""
        buf = np.empty((self.N, self.N))
        self._check(self._lib.gpb200_get_factor(self._h, _as_dp(buf)), "get_factor")
        return buf.T.copy()      # buffer is column-major U == row-major L

    def inverse(self):
        K = np.empty((self.N, self.N))
        self._check(self._lib.gpb200_get_inverse(self._h, _as_dp(K)), "get_inverse")
        return K

    def inverse_diag(self):
        d = np.empty(self.N)
        self._check(self._lib.gpb200_get_inverse_diag(self._h, _as_dp(d)), "get_inverse_diag")
        return d

    def storage_info(self):
        v = (C.c_int64 * 8)()
        self._check(self._lib.gpb200_storage_info(self._h, v, 8), "storage_info")
        return dict(sharded=bool(v[0]), bytes_F=int(v[1]), bytes_G=int(v[2]), rb=int(v[3]), nranks=int(v[4]), rank=int(v[5]),
                    tma=bool(v[6]), bytes_cv=int(v[7]))

    def _own_rows_inverse(self):
        """sharded storage: this rank's rows of K^-1 (lower part valid), zeros elsewhere"""
        K = np.empty((self.N, self.N))
        self._check(self._lib.gpb200_get_inverse(self._h, _as_dp(K)), "get_inverse")
        return np.tril(K)

    def timings(self):
        ms = np.zeros(17)
        self._check(self._lib.gpb200_get_timings(self._h, _as_dp(ms), 17), "get_timings")
        return dict(gram=ms[0], cholesky=ms[1], solve_mll=ms[2], inverse=ms[3], trace=ms[4], predict=ms[5],
                    gemm_launches=ms[6], gemm_ms=ms[7], gemm_flops=ms[8], gpa_scan=ms[9], gpa_product=ms[10],
                    pgrad_crossgram=ms[11], pgrad_trsm=ms[12], pgrad_transpose=ms[13], pgrad_trsm_right=ms[14],
                    pgrad_contract=ms[15], grad_inputs=ms[16])

    def set_stream(self, cuda_stream):
        """Run on the caller's CUDA stream (int handle, e.g. torch.cuda.current_stream().cuda_stream); 0/None = private."""
        self._check(self._lib.gpb200_set_stream(self._h, C.c_void_p(int(cuda_stream) if cuda_stream else None)), "set_stream")

    # -- multi-GPU (one process per GPU) -------------------------------------------------------
    def nccl_unique_id(self):
        buf = C.create_string_buffer(128)
        rc = (self._lib if self is not None else load_library()).gpb200_nccl_unique_id(C.cast(buf, C.c_void_p))
        if rc != OK:
            raise RuntimeError("gpb200_nccl_unique_id failed (%d)" % rc)
        return buf.raw

    def comm_init(self, nranks, rank, id128):
        if len(id128) != 128:
            raise ValueError("NCCL unique id must be 128 bytes")
        ib = C.create_string_buffer(bytes(id128), 128)
        self._check(self._lib.gpb200_comm_init(self._h, int(nranks), int(rank), C.cast(ib, C.c_char_p)), "comm_init")
        self.nranks, self.rank = int(nranks), int(rank)

    IPC_BYTES = 512

    def ipc_export(self):
        buf = C.create_string_buffer(self.IPC_BYTES)
        self._check(self._lib.gpb200_ipc_export(self._h, C.cast(buf, C.c_void_p)), "ipc_export")
        return buf.raw

    def ipc_import(self, blobs):
        """blobs: list of nranks byte strings in rank order (own entry ignored)."""
        joined = b"".join(bytes(b) for b in blobs)
        if len(joined) != self.IPC_BYTES * len(blobs):
            raise ValueError("ipc_import: every blob must be %d bytes" % self.IPC_BYTES)
        buf = C.create_string_buffer(joined, len(joined))
        self._check(self._lib.gpb200_ipc_import(self._h, len(blobs), C.cast(buf, C.c_void_p)), "ipc_import")

    def fp64_peak(self):
        a, b = C.c_double(), C.c_double()
        self._check(self._lib.gpb200_fp64_peak(self._h, C.byref(a), C.byref(b)), "fp64_peak")
        return dict(dmma_tflops=a.value, dfma_tflops=b.value)

    def launch_count(self):
        return int(self._lib.gpb200_launch_count(self._h))

    def dgemm_nt_device(self, impl, M, N, K, alpha, dA, lda, dB, ldb, beta, dC, ldc, lower_only=False, reps=1):
        ms = C.c_double()
        self._check(self._lib.gpb200_dgemm_nt_device(self._h, int(impl), M, N, K, float(alpha), C.c_void_p(dA), lda,
                                                     C.c_void_p(dB), ldb, float(beta), C.c_void_p(dC), ldc,
                                                     1 if lower_only else 0, int(reps), C.byref(ms)), "dgemm_nt")
        return ms.value

    GEMM_DESC_LEN = 79

    def gemm_nt_desc(self, impl, desc, alpha, beta):
        """One NT GEMM launch from the flat descriptor of include/gpb200.h (GPB200_GEMM_DESC_LEN int64)."""
        d = np.ascontiguousarray(desc, dtype=np.int64)
        self._check(self._lib.gpb200_gemm_nt_desc(self._h, int(impl), d.ctypes.data_as(_lp), d.size, float(alpha),
                                                  float(beta)), "gemm_nt_desc")

    def fsa_gemm_items(self, items, alpha_beta):
        """items: (n, 8) int64 rows (C, A, B, ldc, lda, ldb, K, lower); alpha_beta: (n, 2)."""
        it = np.ascontiguousarray(items, dtype=np.int64).reshape(-1, 8)
        ab = np.ascontiguousarray(alpha_beta, dtype=np.float64).reshape(-1, 2)
        if ab.shape[0] != it.shape[0]:
            raise ValueError("fsa_gemm_items: one (alpha, beta) per item")
        self._check(self._lib.gpb200_fsa_gemm_items(self._h, it.ctypes.data_as(_lp), _as_dp(ab), it.shape[0]),
                    "fsa_gemm_items")

    def potrf_tiles(self, mode, args):
        """Diagonal-tile leaf (mode 0: strided tiles, 39 arguments; mode 1: 6 per item).  Returns the device info word."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        info = C.c_int32()
        self._check(self._lib.gpb200_potrf_tiles(self._h, int(mode), a.ctypes.data_as(_lp), a.size, C.byref(info)),
                    "potrf_tiles")
        return int(info.value)

    def trsv_tiles(self, schedule, direction, args):
        """Blocked triangular solve (schedule 0: per block step, 1: single launch; direction 0: L^-1, 1: L^-T) on
        (F, ldf, Dinv or DinvT, rhs, out, Npad).  Returns the watchdog word."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        wd = C.c_int32()
        self._check(self._lib.gpb200_trsv_tiles(self._h, int(schedule), int(direction), a.ctypes.data_as(_lp), a.size,
                                                C.byref(wd)), "trsv_tiles")
        return int(wd.value)

    def gpa_kernels(self, which, args):
        """GPA kernel (0 trmv, 1 trmv_t, 2 scan) on the device buffers of include/gpb200.h."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        self._check(self._lib.gpb200_gpa_kernels(self._h, int(which), a.ctypes.data_as(_lp), a.size), "gpa_kernels")

    def row_reductions(self, which, args):
        """Fixed-order reduction (0 dot, 1 sum, 2 rowdot, 3 rowvar, 4 rowdot2) on the device buffers of include/gpb200.h."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        self._check(self._lib.gpb200_row_reductions(self._h, int(which), a.ctypes.data_as(_lp), a.size), "row_reductions")

    FSA_KERNELS = ("gram", "bdmv", "mask", "permute", "resid", "outer", "trace", "axpy_t", "crossgram", "rowdot", "var",
                   "crossgram_dx", "block_dx")
    FITC_CV_KERNELS = ("delta", "rows", "invdiag", "eblock", "qs", "wvec", "gather", "diag", "colscale", "scale", "fitc_g",
                       "fitc_wfu", "fitc_wuu", "symmetrize", "inducing_dx", "rows_dx")

    def fsa_kernels(self, name, args, fargs=()):
        """One FSA block-diagonal kernel (include/gpb200.h) by name, on device buffers: args = the int64 arguments followed
        by the flattened items, fargs = theta (and diag_add) or alpha."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        f = np.ascontiguousarray(fargs, dtype=np.float64).ravel()
        self._check(self._lib.gpb200_fsa_kernels(self._h, self.FSA_KERNELS.index(name), a.ctypes.data_as(_lp), a.size,
                                                 _as_dp(f), f.size), "fsa_kernels")

    GRAM_KERNELS = ("gram_lower", "crossgram", "gram_full", "kdiag", "gram_grad_full", "crossgram_grad", "trace",
                    "trace_rect", "kdiag_grad", "crossgram_dx", "mirror_lower_tiles", "inputs_dx", "gram_seiso_tma",
                    "trace_seiso_tma")

    def gram_kernels(self, name, args, fargs=()):
        """One dense Gram-family kernel (include/gpb200.h) by name, on device buffers: args = the int64 arguments,
        fargs = theta (and the nugget or c)."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        f = np.ascontiguousarray(fargs, dtype=np.float64).ravel()
        self._check(self._lib.gpb200_gram_kernels(self._h, self.GRAM_KERNELS.index(name), a.ctypes.data_as(_lp), a.size,
                                                  _as_dp(f), f.size), "gram_kernels")

    VEC_KERNELS = ("ew", "spd_from_cov", "add_rowvec", "gather_block")

    def vec_kernels(self, name, args, fargs=()):
        """One elementwise or sampling helper (include/gpb200.h) by name, on device buffers: fargs = s (ew) or the nugget
        (spd_from_cov)."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        f = np.ascontiguousarray(fargs, dtype=np.float64).ravel()
        self._check(self._lib.gpb200_vec_kernels(self._h, self.VEC_KERNELS.index(name), a.ctypes.data_as(_lp), a.size,
                                                 _as_dp(f), f.size), "vec_kernels")

    def fitc_cv_kernels(self, name, args, fargs=()):
        """One sparse cross-validation row kernel or FITC element kernel (include/gpb200.h) by name, on device buffers."""
        a = np.ascontiguousarray(args, dtype=np.int64).ravel()
        f = np.ascontiguousarray(fargs, dtype=np.float64).ravel()
        self._check(self._lib.gpb200_fitc_cv_kernels(self._h, self.FITC_CV_KERNELS.index(name), a.ctypes.data_as(_lp),
                                                     a.size, _as_dp(f), f.size), "fitc_cv_kernels")


class FitcEngine:
    """Owns one gpb200_fitc handle: the FITC sparse strategy (src/sparse/fully_indep_train_conditional.jl)."""

    def __init__(self, device=0):
        self._lib = load_library()
        self._h = _H()
        rc = self._lib.gpb200_fitc_create(C.byref(self._h), int(device))
        if rc != OK:
            msg = self._lib.gpb200_last_error(None)
            raise RuntimeError("gpb200_fitc_create failed (%d): %s" % (rc, msg.decode() if msg else "?"))
        self.N = self.M = self.d = 0

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.gpb200_fitc_destroy(self._h)
            self._h = _H()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc == OK:
            return
        msg = self._lib.gpb200_fitc_last_error(self._h)
        msg = msg.decode() if msg else ""
        if rc > 0:
            raise PosDefException(rc)
        if rc in (EINVAL, ESTATE):
            raise ValueError("%s: %s" % (what, msg))
        raise RuntimeError("%s failed (%d): %s" % (what, rc, msg))

    def set_data(self, x_pm, xu_pm):
        x_pm = np.ascontiguousarray(x_pm, dtype=np.float64)
        xu_pm = np.ascontiguousarray(xu_pm, dtype=np.float64)
        (N, d), (M, d2) = x_pm.shape, xu_pm.shape
        if d != d2:
            raise ValueError("inducing points and inputs must have the same dimension")
        self._check(self._lib.gpb200_fitc_set_data(self._h, N, d, _as_dp(x_pm), d, M, _as_dp(xu_pm), d), "fitc_set_data")
        self.N, self.M, self.d = N, M, d

    def grad_kernel(self):
        g = np.empty(max(self.n_theta, 1))
        self._check(self._lib.gpb200_fitc_grad_kernel(self._h, _as_dp(g)), "fitc_grad_kernel")
        return g[:self.n_theta].copy()

    def grad_kernel_inducing(self, want_kernel=True):
        """one sweep: (dmll_kernel[n_theta] or None, dmll_xu (M, d)); dmll_kernel bitwise grad_kernel's"""
        g = np.empty(max(self.n_theta, 1)) if want_kernel else None
        gx = np.empty((self.M, self.d))
        self._check(self._lib.gpb200_fitc_grad_kernel_inducing(self._h, _as_dp(g) if want_kernel else None, _as_dp(gx)),
                    "fitc_grad_kernel_inducing")
        return (g[:self.n_theta].copy() if want_kernel else None), gx

    def set_inducing(self, xu_pm):
        """replace the inducing points (M, d) in place; factorize + mll must follow"""
        xu_pm = np.ascontiguousarray(xu_pm, dtype=np.float64)
        if xu_pm.shape != (self.M, self.d):
            raise ValueError("fitc_set_inducing: the inducing points must keep their shape (%d, %d)" % (self.M, self.d))
        self._check(self._lib.gpb200_fitc_set_inducing(self._h, self.M, _as_dp(xu_pm), self.d), "fitc_set_inducing")

    def grad_kernel_inputs(self, want_kernel=True, want_inducing=False):
        """one sweep: (dmll_kernel[n_theta] or None, dmll_xu (M, d) or None, dmll_x (N, d)) without the mean's part;
        dmll_kernel and dmll_xu bitwise those of grad_kernel and grad_kernel_inducing"""
        g = np.empty(max(self.n_theta, 1)) if want_kernel else None
        gu = np.empty((self.M, self.d)) if want_inducing else None
        gx = np.empty((self.N, self.d))
        self._check(self._lib.gpb200_fitc_grad_kernel_inputs(self._h, _as_dp(g) if want_kernel else None,
                                                             _as_dp(gu) if want_inducing else None, _as_dp(gx)),
                    "fitc_grad_kernel_inputs")
        return (g[:self.n_theta].copy() if want_kernel else None), gu, gx

    def set_inputs(self, x_pm):
        """replace the training inputs (N, d) in place (FSA keeps its blocks by index); factorize + mll must follow"""
        x_pm = np.ascontiguousarray(x_pm, dtype=np.float64)
        if x_pm.shape != (self.N, self.d):
            raise ValueError("fitc_set_inputs: the inputs must keep their shape (%d, %d)" % (self.N, self.d))
        self._check(self._lib.gpb200_fitc_set_inputs(self._h, self.N, _as_dp(x_pm), self.d), "fitc_set_inputs")

    def append(self, xnew_pm, r_new):
        """append the rows xnew_pm (k, d) with residuals r_new = y - m(x) (k,): (mll, logdet) of the grown data.  Predictions
        work at once; alpha, the gradients and cross-validation need mll(y - m(x)) over all rows first."""
        xnew_pm = np.ascontiguousarray(xnew_pm, dtype=np.float64).reshape(-1, self.d)
        r = np.ascontiguousarray(r_new, dtype=np.float64).ravel()
        if r.size != xnew_pm.shape[0]:
            raise ValueError("fitc_append: %d rows, but %d residuals" % (xnew_pm.shape[0], r.size))
        m, ld = C.c_double(), C.c_double()
        rc = self._lib.gpb200_fitc_append(self._h, r.size, _as_dp(xnew_pm), self.d, _as_dp(r), C.byref(m), C.byref(ld))
        if rc == OK or rc > 0:                                   # a Sigma_QR that is not positive definite keeps the grown data
            self.N += r.size
        self._check(rc, "fitc_append")
        return m.value, ld.value

    def grad_inputs_timings(self):
        """device times (ms) of the last grad_kernel_inputs: the dmll/dX contractions summed, the whole call"""
        out = np.zeros(11)
        self._check(self._lib.gpb200_fitc_get_timings(self._h, _as_dp(out), 11), "fitc_get_timings")
        return out[9:].copy()

    def grad_inducing_timings(self):
        """device times (ms) of the last grad_kernel_inducing: the dmll/dXu contractions summed, the whole call"""
        out = np.zeros(9)
        self._check(self._lib.gpb200_fitc_get_timings(self._h, _as_dp(out), 9), "fitc_get_timings")
        return out[7:].copy()

    def set_kernel(self, ops, dims, n_theta):
        self.n_theta = int(n_theta)
        ops = np.ascontiguousarray(ops, dtype=np.int32).reshape(-1, OP_STRIDE)
        dims = np.ascontiguousarray(dims, dtype=np.int32)
        self._check(self._lib.gpb200_fitc_set_kernel(self._h, ops.shape[0], ops.ctypes.data_as(_ip), dims.size,
                                                     dims.ctypes.data_as(_ip), int(n_theta)), "fitc_set_kernel")

    def factorize(self, theta, log_noise):
        theta = np.ascontiguousarray(theta, dtype=np.float64)
        self._check(self._lib.gpb200_fitc_factorize(self._h, _as_dp(theta), float(log_noise)), "fitc_factorize")

    def mll(self, y_minus_mean):
        r = np.ascontiguousarray(y_minus_mean, dtype=np.float64)
        if r.shape != (self.N,):
            raise ValueError("fitc_mll: y must have length N")
        alpha = np.empty(self.N)
        m, ld = C.c_double(), C.c_double()
        self._check(self._lib.gpb200_fitc_mll(self._h, _as_dp(r), _as_dp(alpha), C.byref(m), C.byref(ld)), "fitc_mll")
        return alpha, m.value, ld.value

    def grad_noise(self):
        g = C.c_double()
        self._check(self._lib.gpb200_fitc_grad_noise(self._h, C.byref(g)), "fitc_grad_noise")
        return g.value

    def predict(self, xs_pm, want_var=True):
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        Ms, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        mu = np.empty(Ms)
        var = np.empty(Ms) if want_var else None
        self._check(self._lib.gpb200_fitc_predict(self._h, Ms, _as_dp(xs_pm), d, _as_dp(mu),
                                                  _as_dp(var) if want_var else None), "fitc_predict")
        return mu, var

    def predict_grad(self, xs_pm, alpha=None, want_var=True):
        """as Engine.predict_grad: (mu_minus_mean, var or None, dmu (Ms, d), dvar (Ms, d) or None); alpha must be None (the
        sparse engine's own u is used)"""
        if alpha is not None:
            raise ValueError("fitc_predict_grad: the sparse engine predicts from its own u")
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        Ms, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        mu, dmu = np.empty(Ms), np.empty((Ms, d))
        var = np.empty(Ms) if want_var else None
        dvar = np.empty((Ms, d)) if want_var else None
        self._check(self._lib.gpb200_fitc_predict_grad(self._h, Ms, _as_dp(xs_pm), d, _as_dp(mu), _as_dp(var) if want_var else None,
                                                       _as_dp(dmu), _as_dp(dvar) if want_var else None), "fitc_predict_grad")
        return mu, var, dmu, dvar

    def comm_init(self, nranks, rank, id128):
        ib = C.create_string_buffer(bytes(id128), 128)
        self._check(self._lib.gpb200_fitc_comm_init(self._h, int(nranks), int(rank), C.cast(ib, C.c_char_p)), "fitc_comm_init")

    def predict_cov(self, xs_pm):
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        Ms, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        mu = np.empty(Ms)
        cov = np.empty((Ms, Ms))
        self._check(self._lib.gpb200_fitc_predict_cov(self._h, Ms, _as_dp(xs_pm), d, _as_dp(mu), _as_dp(cov)), "fitc_predict_cov")
        return mu, cov

    def set_mode(self, mode):
        """0 FITC, 1 DTC, 2 SoR, 3 FSA."""
        self._check(self._lib.gpb200_fitc_set_mode(self._h, int(mode)), "fitc_set_mode")

    def set_blocks(self, block_ptr, idx):
        """FSA training blocks in CSR form (0-based): block b is idx[block_ptr[b]:block_ptr[b+1]]."""
        block_ptr = np.ascontiguousarray(block_ptr, dtype=np.int64)
        idx = np.ascontiguousarray(idx, dtype=np.int64)
        if block_ptr.ndim != 1 or block_ptr.size < 2 or idx.shape != (self.N,):
            raise ValueError("fitc_set_blocks: block_ptr must have nblocks + 1 >= 2 entries and idx N entries")
        self._check(self._lib.gpb200_fitc_set_blocks(self._h, block_ptr.size - 1, block_ptr.ctypes.data_as(_lp),
                                                     idx.ctypes.data_as(_lp)), "fitc_set_blocks")

    def predict_fsa(self, xs_pm, block_of, want_var=True, full_cov=False):
        """FSA predictions: block_of[i] = training block paired with test point i (-1: none).  Returns (mu, var or cov)."""
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        Ms, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        block_of = np.ascontiguousarray(block_of, dtype=np.int64)
        if block_of.shape != (Ms,):
            raise ValueError("fitc_predict_fsa: block_of must have one entry per test point")
        mu = np.empty(Ms)
        var = np.empty(Ms) if (want_var and not full_cov) else None
        cov = np.empty((Ms, Ms)) if full_cov else None
        self._check(self._lib.gpb200_fitc_predict_fsa(self._h, Ms, _as_dp(xs_pm), d, block_of.ctypes.data_as(_lp), _as_dp(mu),
                                                      _as_dp(var) if var is not None else None,
                                                      _as_dp(cov) if cov is not None else None), "fitc_predict_fsa")
        return mu, (cov if full_cov else var)

    def predict_fsa_grad(self, xs_pm, block_of, want_var=True):
        """FSA predictions and their gradients with respect to the test inputs: (mu_minus_mean, var or None, dmu (Ms, d),
        dvar (Ms, d) or None), mu and var bitwise those of predict_fsa."""
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        Ms, d = xs_pm.shape
        if d != self.d:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        block_of = np.ascontiguousarray(block_of, dtype=np.int64)
        if block_of.shape != (Ms,):
            raise ValueError("fitc_predict_fsa_grad: block_of must have one entry per test point")
        mu, dmu = np.empty(Ms), np.empty((Ms, d))
        var = np.empty(Ms) if want_var else None
        dvar = np.empty((Ms, d)) if want_var else None
        self._check(self._lib.gpb200_fitc_predict_fsa_grad(self._h, Ms, _as_dp(xs_pm), d, block_of.ctypes.data_as(_lp),
                                                           _as_dp(mu), _as_dp(var) if want_var else None, _as_dp(dmu),
                                                           _as_dp(dvar) if want_var else None), "fitc_predict_fsa_grad")
        return mu, var, dmu, dvar

    # -- cross-validation (modes 0-2, one GPU; after factorize + mll) ---------------------------------------------------
    def inverse_diag(self):
        """diag(Sigma^-1)[N]."""
        d = np.empty(self.N)
        self._check(self._lib.gpb200_fitc_get_inverse_diag(self._h, _as_dp(d)), "fitc_get_inverse_diag")
        return d

    def cv_param(self, param, alpha=None):
        """(Z_j alpha, diag(Z_j Sigma^-1)) for kernel parameter `param` (index into the full parameter vector) or -1 = noise."""
        za, dg = np.empty(self.N), np.empty(self.N)
        ap = _as_dp(np.ascontiguousarray(alpha, dtype=np.float64)) if alpha is not None else None
        self._check(self._lib.gpb200_fitc_cv_param(self._h, int(param), ap, _as_dp(za), _as_dp(dg)), "fitc_cv_param")
        return za, dg

    def cv_block(self, which, idx):
        """Sigma^-1[V,V] (which 0) or (Z_j Sigma^-1)[V,V] of the last cv_param (which 1)."""
        idx = np.ascontiguousarray(idx, dtype=np.int64)
        out = np.empty((idx.size, idx.size))
        self._check(self._lib.gpb200_fitc_cv_block(self._h, int(which), idx.size, idx.ctypes.data_as(C.POINTER(C.c_int64)),
                                                   _as_dp(out)), "fitc_cv_block")
        return out

    def rand(self, xs_pm, z, nugget=1e-10, block_of=None):
        """z: (nsamp, Ms) standard-normal draws (== Julia's Ms x nsamp column-major); block_of[Ms] in FSA mode only (as in
        predict_fsa).  Returns (mu_minus_mean[Ms], samples (nsamp, Ms))."""
        xs_pm = np.ascontiguousarray(xs_pm, dtype=np.float64)
        z = np.ascontiguousarray(z, dtype=np.float64)
        Ms, d = xs_pm.shape
        if d != self.d or z.ndim != 2 or z.shape[1] != Ms:
            raise ValueError("fitc_rand: inconsistent dimensions")
        bp = None
        if block_of is not None:
            block_of = np.ascontiguousarray(block_of, dtype=np.int64)
            if block_of.shape != (Ms,):
                raise ValueError("fitc_rand: block_of must have one entry per test point")
            bp = block_of.ctypes.data_as(_lp)
        mu = np.empty(Ms)
        out = np.empty_like(z)
        self._check(self._lib.gpb200_fitc_rand(self._h, Ms, _as_dp(xs_pm), d, bp, z.shape[0], _as_dp(z), float(nugget),
                                               _as_dp(mu), _as_dp(out)), "fitc_rand")
        return mu, out

    def rand_timings(self):
        """device times (ms) of the last rand: Sigma* build, make_posdef! + Cholesky, unwhiten! + mu"""
        out = np.zeros(3)
        self._check(self._lib.gpb200_fitc_get_timings(self._h, _as_dp(out), 3), "fitc_get_timings")
        return out

    def predict_fsa_grad_timings(self):
        """device times (ms) of the last predict_fsa_grad, summed over its test chunks: predict_fsa's launches, s and the
        second block sweep, the K_uu^-1 TRSMs, the contraction"""
        out = np.zeros(7)
        self._check(self._lib.gpb200_fitc_get_timings(self._h, _as_dp(out), 7), "fitc_get_timings")
        return out[3:].copy()

    def launch_count(self):
        return int(self._lib.gpb200_fitc_launch_count(self._h))


class LocalGroupEngine:
    """R engines on ONE device acting as the R ranks of the ROW-SHARDED multi-GPU schedules (gpb200_group_create,
    csrc/shard_impl.cuh): each virtual rank maps only its own block rows of the N x N factor / inverse, collectives are
    event-ordered device copies.  Same interface as `Engine`, so `GPE(..., engine=LocalGroupEngine(4))` runs the whole
    host mirror over the sharded storage on a single GPU (tests; the production path is one process per GPU + NCCL)."""

    def __init__(self, nranks, device=0, rb=0):
        self.engines = [Engine(device) for _ in range(int(nranks))]
        self.lead = self.engines[0]
        arr = (_H * len(self.engines))(*[e._h for e in self.engines])
        rc = self.lead._lib.gpb200_group_create(arr, len(self.engines))
        self.lead._check(rc, "group_create")
        self.nranks = len(self.engines)
        if rb:
            self.set_option("shard_rb", rb)

    # replicated state: every virtual rank gets it
    def set_data(self, x_pm):
        for e in self.engines:
            e.set_data(x_pm)
        self.N, self.d = self.lead.N, self.lead.d

    def set_kernel(self, ops, dims, n_theta):
        for e in self.engines:
            e.set_kernel(ops, dims, n_theta)
        self.n_theta = self.lead.n_theta

    def set_option(self, key, value):
        for e in self.engines:
            e.set_option(key, value)

    def close(self):
        for e in self.engines:
            e.close()

    # collective entry points: the leader drives every rank
    def factorize(self, *a, **k):
        return self.lead.factorize(*a, **k)

    def mll(self, *a, **k):
        return self.lead.mll(*a, **k)

    def solve(self, *a, **k):
        return self.lead.solve(*a, **k)

    def logdet(self):
        return self.lead.logdet()

    def grad_prepare(self):
        return self.lead.grad_prepare()

    def grad_kernel(self, *a, **k):
        return self.lead.grad_kernel(*a, **k)

    def grad_inputs(self, *a, **k):
        return self.lead.grad_inputs(*a, **k)

    def predict(self, *a, **k):
        return self.lead.predict(*a, **k)

    def rand(self, *a, **k):
        return self.lead.rand(*a, **k)

    def predict_grad(self, *a, **k):
        return self.lead.predict_grad(*a, **k)

    def cv_param(self, *a, **k):
        return self.lead.cv_param(*a, **k)

    def cv_block(self, *a, **k):
        return self.lead.cv_block(*a, **k)

    def inverse_diag(self):
        return self.lead.inverse_diag()

    def append(self, xnew_pm):
        """the leader extends every rank's inputs and the distributed factor (ElasticGPE append!)"""
        self.lead.append(xnew_pm)
        for e in self.engines[1:]:
            e.N = self.lead.N
        self.N = self.lead.N

    def timings(self):
        return self.lead.timings()

    def launch_count(self):
        return sum(e.launch_count() for e in self.engines)

    def gram(self):
        return self.lead.gram()

    # debug getters: every rank returns its own rows (zeros elsewhere); the pieces add up to the full matrix
    def factor_upper(self):
        return sum(e.factor_upper() for e in self.engines)

    def inverse(self):
        K = sum(e._own_rows_inverse() for e in self.engines)
        return np.tril(K) + np.tril(K, -1).T
