"""GPA -- host-side mirror of the reference's GP with a non-Gaussian likelihood (src/GPA.jl).  The latent function is
whitened, f = L v + mu with L L' = K (v ~ N(0, I)); the target is log p(y | f) - (v'v + N log 2pi) / 2.

The device holds the factor and does the O(N^2) / O(N^3) work: gpb200_unwhiten (f = L v) and gpb200_gpa_grad (L' dl_df and
the kernel gradient through the Cholesky factor, src/GPA.jl:130-173).  The likelihood and the mean stay on the host (O(N)).
Gradient order [v; lik; mean; kernel] (GPA.jl:183-228), with -v from the N(0, I) prior on v; no hyper-parameter priors, as
in the GPE mirror."""
import math

import numpy as np

from . import capi
from .gpe import _as_dxn, _predict_f_grad
from .kernels import Kernel, flatten
from .likelihoods import Likelihood
from .means import Mean, MeanZero

_LOG2PI = math.log(2.0 * math.pi)
_NO_NOISE = -400.0          # exp(2 * -400) == 0.0: the Gram diagonal gets only the explicit nugget


class GPA:
    def __init__(self, x, y, mean=None, kernel=None, lik=None, device=0, engine=None):
        if kernel is None or not isinstance(kernel, Kernel):
            raise ValueError("GPA needs a kernel")
        if lik is None or not isinstance(lik, Likelihood):
            raise ValueError("GPA needs a likelihood")
        self.mean = mean if mean is not None else MeanZero()
        if not isinstance(self.mean, Mean):
            raise ValueError("mean must be a Mean")
        self.kernel, self.lik = kernel, lik
        x = _as_dxn(x)
        y = lik.check_y(y)
        if x.shape[1] != y.size:
            raise ValueError("Input and output observations must have consistent dimensions.")     # GPA.jl:45
        self.x, self.y = x, y
        self.dim, self.nobs = x.shape
        self._xpm = np.ascontiguousarray(x.T)
        self._eng = engine if engine is not None else capi.Engine(device)
        self._eng.set_data(self._xpm)
        ops, dims, theta, exposed = flatten(self.kernel, self.dim)
        self._exposed = exposed
        self._eng.set_kernel(ops, dims, theta.size)
        self.v = np.zeros(self.nobs)                  # GPA.jl:47
        self.mu = None
        self.ll = float("nan")
        self.target = float("nan")
        self.dll = None
        self.dtarget = None
        self.initialise_target()

    @property
    def μ(self):
        return self.mu

    # ---- log target ----------------------------------------------------------------------
    def _f(self):
        return self._eng.unwhiten(self.v) + self.mu                    # unwhiten(gp.cK, gp.v) + gp.μ

    def initialise_ll(self):
        """initialise_ll!(gp) (GPA.jl:101-109): cK = PDMat(Σ + 1e-6 I)."""
        self.mu = self.mean.mean(self._xpm)
        self._eng.factorize(flatten(self.kernel, self.dim)[2], _NO_NOISE, extra_nugget=1e-6)
        self.ll = float(np.sum(self.lik.log_dens(self._f(), self.y)))
        return self

    def update_cK(self):
        """update_cK!(gp::GPA) (GPA.jl:111-114): Gram + exp(2 * -20) nugget + Cholesky on the device."""
        self._eng.factorize(flatten(self.kernel, self.dim)[2], -20.0)
        self._inputs_moved = False

    def update_ll(self, process=True, lik=True, domean=True, kern=True, inputs=False):
        """update_ll!(gp) (GPA.jl:118-128).  After set_params(..., inputs=True) the factor is refreshed whatever kern says."""
        if kern or getattr(self, "_inputs_moved", False):
            self.update_cK()
        self.mu = self.mean.mean(self._xpm)
        self.ll = float(np.sum(self.lik.log_dens(self._f(), self.y)))
        return self

    def _prior_v(self):
        return -(float(self.v @ self.v) + _LOG2PI * self.nobs) / 2.0

    def initialise_target(self):                                        # GPA.jl:245-250
        self.initialise_ll()
        self.target = self.ll + self._prior_v()
        return self

    def update_target(self, process=True, lik=True, domean=True, kern=True, inputs=False):      # GPA.jl:261-266
        self.update_ll(process=process, lik=lik, domean=domean, kern=kern)
        self.target = self.ll + self._prior_v()
        return self

    def update_dll(self, process=True, lik=True, domean=True, kern=True, inputs=False):
        """update_dll!(gp, precomp) (GPA.jl:183-228): [L' dl_df; sum dlog_dens_dθ; dmll_mean!; dll_kern!].  inputs=True (not
        in the reference) appends dll/dX as vec(X): sum_j S_ij dk(x_i, x_j)/dx_i over the S that the kernel gradient forms on
        the device, plus (dl_df)_i dm(x_i)/dx_i."""
        f = self._f()                                                   # precompute! (GPA.jl:158-163)
        dl_df = self.lik.dlog_dens_df(f, self.y)
        u, gk = None, None
        if process or kern or inputs:
            u, gk = self._eng.gpa_grad(self.v, dl_df, process=process, kern=kern or inputs)
        out = []
        if process:
            out.extend(u)
        if lik and self.lik.num_params() > 0:
            out.extend(np.sum(self.lik.dlog_dens_dtheta(f, self.y), axis=0))
        if domean and self.mean.num_params() > 0:
            out.extend(self.mean.grad_stack(self._xpm).T @ dl_df)
        if kern:
            out.extend(gk[self._exposed])                               # FixedKernel selection, fixed_kernel.jl:64-66
        if inputs:
            out.extend((self._eng.grad_inputs() + dl_df[:, None] * self.mean.grad_x(self._xpm)).ravel())
        self.dll = np.array(out, dtype=np.float64)
        return self

    def update_dtarget(self, **kw):                                     # GPA.jl:268-272
        self.update_dll(**kw)
        self.dtarget = self.dll.copy()
        if kw.get("process", True):
            self.dtarget[:self.nobs] -= self.v                          # prior_gradlogpdf: -v (GPA.jl:384-385)
        return self

    def update_target_and_dtarget(self, **kw):                          # GPA.jl:283-291
        self.update_target(**kw)
        self.update_dtarget(**kw)
        return self

    # ---- parameters ----------------------------------------------------------------------
    def get_params(self, lik=True, domean=True, kern=True, inputs=False):             # GPA.jl:336-349
        """inputs=True (not in the reference) appends vec(X), one point after another."""
        p = list(self.v)
        if lik and self.lik.num_params() > 0:
            p.extend(self.lik.get_params())
        if domean and self.mean.num_params() > 0:
            p.extend(self.mean.get_params())
        if kern:
            p.extend(self.kernel.get_params())
        if inputs:
            p.extend(self._xpm.ravel())
        return np.array(p, dtype=np.float64)

    def num_params(self, lik=True, domean=True, kern=True, inputs=False):             # GPA.jl:351-357
        n = self.nobs + (self.dim * self.nobs if inputs else 0)
        if lik:
            n += self.lik.num_params()
        if domean:
            n += self.mean.num_params()
        if kern:
            n += self.kernel.num_params()
        return n

    def set_params(self, hyp, process=True, lik=True, domean=True, kern=True, inputs=False):     # GPA.jl:359-381
        """inputs=True: the last dim * nobs entries are vec(X), uploaded in place; the next update_ll refactorises."""
        hyp = np.asarray(hyp, dtype=np.float64)
        if inputs:
            nx = self.dim * self.nobs
            if hyp.size < nx:
                raise ValueError("wrong number of parameters")
            self.set_params(hyp[:hyp.size - nx], process=process, lik=lik, domean=domean, kern=kern)
            xpm = np.ascontiguousarray(hyp[hyp.size - nx:].reshape(self.nobs, self.dim))
            self._eng.set_data(xpm)
            self._xpm, self.x = xpm, xpm.T
            self._inputs_moved = True
            return self
        i = 0
        if process:
            self.v = hyp[:self.nobs].copy()
            i += self.nobs
        n = self.lik.num_params()
        if lik and n > 0:
            self.lik.set_params(list(hyp[i:i + n]))
            i += n
        n = self.mean.num_params()
        if domean and n > 0:
            self.mean.set_params(hyp[i:i + n])
            i += n
        if kern:
            n = self.kernel.num_params()
            self.kernel.set_params(list(hyp[i:i + n]))
            i += n
        if i != hyp.size:
            raise ValueError("wrong number of parameters")
        return self

    # ---- prediction ----------------------------------------------------------------------
    def _alpha(self):
        return self._eng.solve(self._eng.unwhiten(self.v))            # gp.cK \\ unwhiten(gp.cK, gp.v)  (GPA.jl:294)

    def _xs(self, x):
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        return np.ascontiguousarray(x.T)

    def predict_f(self, x, full_cov=False):
        """predict_f(gp::GPA, x; full_cov) (GP.jl:64-79 through predict_full, GPA.jl:294), batched on the device."""
        xs = self._xs(x)
        mu, var, cov = self._eng.predict(xs, self._alpha(), want_var=not full_cov, full_cov=full_cov)
        mu = mu + self.mean.mean(xs)
        if full_cov:
            return mu, cov
        return mu, np.maximum(var, 0.0)                                 # GP.jl:75

    def predict_f_grad(self, x):
        """predict_f(gp, x) and its gradients with respect to the test inputs: (mu, s2, dmu, ds2), as GPE.predict_f_grad, with
        alpha = K^-1 L v."""
        return _predict_f_grad(self._eng, self._xs(x), self._alpha(), self.mean)

    def predict_y(self, x):
        """predict_y(gp::GPA, x) (GPA.jl:303-306): predict_obs(lik, predict_f(gp, x)...) -- means and variances."""
        mu, s2 = self.predict_f(x)
        return self.lik.predict_obs(mu, s2)

    def rand(self, x, n=1, nugget=1e-10, rng=None):
        """rand(gp, X, n) (GP.jl:120-146) of the latent process: n posterior draws at the columns of x on the device, with
        alpha = K^-1 L v.  Returns a (npred, n) array."""
        rng = np.random.default_rng() if rng is None else rng
        xs = self._xs(x)
        z = rng.standard_normal((int(n), xs.shape[0]))
        _, draws = self._eng.rand(xs, z, nugget=nugget, alpha=self._alpha())
        return (draws + self.mean.mean(xs)[None, :]).T
