"""FITC -- host mirror of the reference's sparse strategy `FITC(x, Xu, y, mean, kern, logNoise)`
(src/sparse/fully_indep_train_conditional.jl:335-338 == GPE(..., FullyIndepStrat(Xu))), over the
gpb200_fitc_* entry points: update_cK!, alpha / mll / logdet, dmll_noise, dmll_mean!, dmll_kern!,
predict_f / predict_y, rand, and GPE's parameter protocol (get_params / set_params / update_target* / optimize).
DTC, SoR and FSA are modes of the same engine."""
import math

import numpy as np

from . import capi
from .gpe import GPE, _RejectedStep, _as_dxn, _predict_f_grad
from .kernels import flatten
from .means import MeanZero


class FITC:
    _mode = 0

    def __init__(self, x, Xu, y, mean=None, kernel=None, logNoise=-2.0, device=0, distributed=False):
        """distributed=True (one process per GPU, torch.distributed initialised): x / y are THIS rank's slice of the observations,
        Xu / kernel / logNoise are the same everywhere; mll and the gradients are those of the full data set, alpha is the
        slice's."""
        self.mean = mean if mean is not None else MeanZero()
        self.kernel = kernel
        self.logNoise = float(logNoise)
        self.x = _as_dxn(x)
        self.Xu = _as_dxn(Xu)                       # inducing points, dim x M (one point per column)
        self.y = np.asarray(y, dtype=np.float64).ravel()
        self.dim, self.nobs = self.x.shape
        if self.Xu.shape[0] != self.dim or self.y.size != self.nobs:
            raise ValueError("Input and output observations must have consistent dimensions.")
        self._xpm = np.ascontiguousarray(self.x.T)
        self._distributed = bool(distributed)
        self._eng = capi.FitcEngine(device)
        if distributed:
            import torch.distributed as dist
            from .dist import broadcast_bytes
            uid = broadcast_bytes(capi.Engine.nccl_unique_id(None) if dist.get_rank() == 0 else None, src=0)
            self._eng.comm_init(dist.get_world_size(), dist.get_rank(), uid)
        self._eng.set_mode(self._mode)
        self._eng.set_data(self._xpm, np.ascontiguousarray(self.Xu.T))
        ops, dims, theta, exposed = flatten(kernel, self.dim)
        self._exposed = exposed
        self._eng.set_kernel(ops, dims, theta.size)
        self.alpha = None
        self.mll = float("nan")
        self.dmll = None
        self.update_mll()

    def update_mll(self, noise=True, domean=True, kern=True):
        """update_mll! (src/GPE.jl:202-212) with cK::FullyIndepPDMat.  The flags are GPE's (update_target passes them);
        the sparse factorisation is rebuilt whatever they say."""
        self._eng.factorize(flatten(self.kernel, self.dim)[2], self.logNoise)
        mu = self.mean.mean(self._xpm)
        self.alpha, self.mll, self.logdet = self._eng.mll(self.y - mu)
        self.target = self.mll
        return self

    def append(self, x, y):
        """append!(gp, x, y) for the sparse strategies (GPEelastic.jl:13-22 has it for the dense model only): add
        observations keeping the hyper-parameters and the inducing points.  The device adds the new rows' rank-k term to
        Sigma_QR and refactors it, O(k M^2 + M^3) whatever nobs is, and returns the mll of the grown data; mll and target are
        set from it.  predict_f, predict_y, predict_f_grad and rand work at once.  alpha is None until the next update_mll,
        which the gradient and cross-validation methods call first when they need it.  On a distributed model x / y are
        this rank's new observations; the call is collective and a rank may pass none."""
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Input observations must have the same dimension as the GP")
        y = np.atleast_1d(np.asarray(y, dtype=np.float64)).ravel()
        if x.shape[1] != y.size:
            raise ValueError("%d observations, but %d targets." % (x.shape[1], y.size))        # GPEelastic.jl:15
        xpm = np.ascontiguousarray(x.T)
        try:
            self.mll, self.logdet = self._eng.append(xpm, y - self.mean.mean(xpm))
        except capi.PosDefException:                              # the device keeps the grown data; update_mll refits it
            self.mll = self.target = float("nan")
            raise
        finally:
            if self._eng.N == self.nobs + y.size:
                self.x = np.concatenate([self.x, x], axis=1)
                self.y = np.concatenate([self.y, y])
                self.nobs = self.y.size
                self._xpm = np.ascontiguousarray(self.x.T)
                self.alpha = None
        self.target = self.mll
        return self

    def _need_alpha(self):
        """alpha of the current data: after append it is refreshed by update_mll (factorize + mll)"""
        if self.alpha is None:
            self.update_mll()

    def update_dmll_noise_mean(self):
        """[dmll_noise (fitc.jl:243-257); dmll_mean! (GPE.jl:282-288)] -- kernel part not built yet."""
        self._need_alpha()
        out = [self._eng.grad_noise()]
        if self.mean.num_params() > 0:
            out.extend(self.mean.grad_stack(self._xpm).T @ self.alpha)
        self.dmll = np.array(out)
        return self

    def update_dmll(self, noise=True, domean=True, kern=True, inducing=False, inputs=False):
        """update_dmll! (src/GPE.jl:298-324) with the FITC strategy: [noise; mean; kernel].  inducing=True appends
        dmll/dXu as vec(Xu) (one point after another); inputs=True then appends dmll/dX as vec(X) (on a distributed model:
        this rank's points), the device's part plus alpha_i dm(x_i)/dx_i.  The kernel part and the point gradients come from
        one device sweep."""
        self._need_alpha()
        out = []
        if noise:
            out.append(self._eng.grad_noise())                                   # fitc.jl:243-257
        if domean and self.mean.num_params() > 0:
            out.extend(self.mean.grad_stack(self._xpm).T @ self.alpha)           # GPE.jl:282-288
        if inputs:
            gk, gu, gx = self._eng.grad_kernel_inputs(want_kernel=kern, want_inducing=inducing)
            if kern:
                out.extend(gk[self._exposed])
            if inducing:
                out.extend(gu.ravel())
            out.extend((gx + self.alpha[:, None] * self.mean.grad_x(self._xpm)).ravel())
        elif inducing:
            gk, gx = self._eng.grad_kernel_inducing(want_kernel=kern)
            if kern:
                out.extend(gk[self._exposed])
            out.extend(gx.ravel())
        elif kern:
            out.extend(self._eng.grad_kernel()[self._exposed])                   # fitc.jl:200-234 + sor.jl:219-253
        self.dmll = np.array(out)
        return self

    def update_mll_and_dmll(self, noise=True, domean=True, kern=True, inducing=False, inputs=False):
        self.update_mll()
        return self.update_dmll(noise=noise, domean=domean, kern=kern, inducing=inducing, inputs=inputs)

    # ---- GPE's parameter protocol, [noise; mean; kernel] (src/GPE.jl:346-510), and optimize! (src/optimize.jl) -----------
    # logNoise is a scalar here; FixedKernel parameters are neither returned nor set, their gradients are dropped
    # (update_dmll's `_exposed`), exactly as for GPE.  inducing=True (not in the reference) appends vec(Xu), Julia's
    # column-major vec of the dim x M matrix, and inputs=True vec(X) of the dim x nobs matrix: [noise; mean; kernel; Xu; X].
    def get_params(self, noise=True, domean=True, kern=True, inducing=False, inputs=False):
        p = [GPE.get_params(self, noise=noise, domean=domean, kern=kern)]
        if inducing:
            p.append(self.Xu.T.ravel())
        if inputs:
            p.append(self._xpm.ravel())
        return np.concatenate(p)

    num_params = GPE.num_params

    def set_params(self, hyp, noise=True, domean=True, kern=True, inducing=False, inputs=False):
        """inducing / inputs: the trailing vec(Xu) / vec(X) are moved on the engine in place (same sizes; FSA keeps its
        blocks by index); the next update_mll refactorises."""
        if not inducing and not inputs:
            return GPE.set_params(self, hyp, noise=noise, domean=domean, kern=kern)
        hyp = np.asarray(hyp, dtype=np.float64)
        nu = self.Xu.size if inducing else 0
        nx = self.x.size if inputs else 0
        if hyp.size != self.num_params(noise=noise, domean=domean, kern=kern, inducing=inducing, inputs=inputs):
            raise ValueError("wrong number of hyper-parameters")
        n0 = hyp.size - nu - nx
        GPE.set_params(self, hyp[:n0], noise=noise, domean=domean, kern=kern)
        if inducing:
            xu_pm = hyp[n0:n0 + nu].reshape(self.Xu.shape[1], self.dim)
            self._eng.set_inducing(xu_pm)
            self.Xu = np.ascontiguousarray(xu_pm.T)
        if inputs:
            xpm = np.ascontiguousarray(hyp[n0 + nu:].reshape(self.nobs, self.dim))
            self._eng.set_inputs(xpm)
            self._xpm, self.x = xpm, xpm.T
        return self

    initialise_target = GPE.initialise_target
    update_target = GPE.update_target

    def update_target_and_dtarget(self, noise=True, domean=True, kern=True, inducing=False, inputs=False):
        return GPE.update_target_and_dtarget(self, noise=noise, domean=domean, kern=kern, inducing=inducing, inputs=inputs)

    def optimize(self, noise=True, domean=True, kern=True, inducing=False, inputs=False, maxiter=100, **kw):
        """optimize!(gp) as GPE.optimize; inducing=True also moves the inducing points (Snelson & Ghahramani's
        pseudo-inputs) and inputs=True the training inputs, with the same exception filter: a step that makes K_uu,
        Sigma_QR or an FSA block singular (PosDefException) is rejected and the parameters, Xu and X included, are rolled
        back.  inputs=True is refused on a distributed model: each rank holds only its own slice of X."""
        if inputs and self._distributed:
            raise ValueError("optimize(inputs=True) needs every training input in one parameter vector; a distributed model "
                             "holds only this rank's slice")
        if not inducing and not inputs:
            return GPE.optimize(self, noise=noise, domean=domean, kern=kern, maxiter=maxiter, **kw)
        from scipy.optimize import minimize

        flags = dict(noise=noise, domean=domean, kern=kern, inducing=inducing, inputs=inputs)
        best = {"f": None}

        def fg(hyp):
            prev = self.get_params(**flags)
            try:
                if not np.all(np.isfinite(hyp)):
                    raise _RejectedStep("non-finite hyper-parameter")
                self.set_params(hyp, **flags)
                self.update_target_and_dtarget(**flags)
                best["f"] = -self.target if best["f"] is None else min(best["f"], -self.target)
                return -self.target, -self.dtarget
            except (np.linalg.LinAlgError, _RejectedStep):            # as GPE.optimize
                self.set_params(prev, **flags)
                return 1e10 + 1e6 * abs(best["f"] or 0.0), np.asarray(hyp, dtype=np.float64) - prev

        res = minimize(fg, self.get_params(**flags), jac=True, method="L-BFGS-B", options=dict(maxiter=maxiter), **kw)
        self.set_params(res.x, **flags)
        self.update_target()
        return res

    # rand(gp, X, n) (src/GP.jl:120-146): GPE's host side; the engine builds Sigma* = predict_f(x; full_cov=true)'s
    # covariance on the device and factors it there.  Returns a (npred, n) array.
    rand = GPE.rand

    def noise_variance(self):
        return math.exp(2.0 * self.logNoise)

    def predict_f(self, x, full_cov=False):
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        xs = np.ascontiguousarray(x.T)
        if full_cov:                                                   # predict_full -> predictMVN (fitc.jl:324-332)
            mu, cov = self._eng.predict_cov(xs)
            return mu + self.mean.mean(xs), cov
        mu, var = self._eng.predict(xs)
        return mu + self.mean.mean(xs), np.maximum(var, 0.0)          # GP.jl:75

    def predict_f_grad(self, x):
        """predict_f(gp, x) and its gradients with respect to the test inputs, (mu, s2, dmu, ds2) as GPE.predict_f_grad"""
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        return _predict_f_grad(self._eng, np.ascontiguousarray(x.T), None, self.mean)

    def predict_y(self, x, full_cov=False):
        mu, s2 = self.predict_f(x, full_cov=full_cov)
        if full_cov:
            return mu, s2 + self.noise_variance() * np.eye(s2.shape[0])       # GPE.jl:412 (ScalMat)
        return mu, s2 + self.noise_variance()

    # ---- cross-validation (src/crossvalidation.jl with cK the sparse covariance) ----------------------------------------
    # GPE's host assembly, unchanged: the engine's inverse_diag / cv_param / cv_block stream the N rows against the M x M
    # inverses instead of reading a resident N x N inverse.
    def _cv_prepare(self):
        """the sparse engine's CV entry points prepare their own M x M inverses; alpha must be that of the current data"""
        self._need_alpha()

    predict_LOO = GPE.predict_LOO
    logp_LOO = GPE.logp_LOO
    _loo_component = GPE._loo_component
    dlogp_LOO = GPE.dlogp_LOO
    predict_CVfold = GPE.predict_CVfold
    logp_CVfold = GPE.logp_CVfold
    _fold_component = GPE._fold_component
    dlogp_CVfold = GPE.dlogp_CVfold


class DTC(FITC):
    """Deterministic Training Conditional (src/sparse/determ_train_conditional.jl): SoR likelihood, FITC-style
    predictive variance."""
    _mode = 1


class SoR(FITC):
    """Subset of Regressors (src/sparse/subsetofregressors.jl)."""
    _mode = 2


FSA_MAX_BLOCK = 2048


def blocks_to_csr(blockindices, nobs):
    """0-based index arrays -> (block_ptr, idx); ValueError unless the blocks partition 0..nobs-1 (empty blocks are allowed)
    and every block holds at most FSA_MAX_BLOCK points."""
    blocks = [np.asarray(b, dtype=np.int64).ravel() for b in blockindices]
    if not blocks:
        raise ValueError("FSA needs at least one block")
    sizes = np.array([b.size for b in blocks], dtype=np.int64)
    if sizes.max() > FSA_MAX_BLOCK:
        raise ValueError("an FSA block holds %d points; at most %d are supported" % (sizes.max(), FSA_MAX_BLOCK))
    idx = np.concatenate(blocks) if sizes.sum() else np.zeros(0, dtype=np.int64)
    if idx.size != nobs or not np.array_equal(np.sort(idx), np.arange(nobs)):
        raise ValueError("the FSA blocks must partition the training points 0..%d" % (nobs - 1))
    block_ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return block_ptr, idx


class FSA(FITC):
    """Full Scale Approximation (src/sparse/full_scale_approximation.jl:480-484): `FSA(x, Xu, blockindices, y, mean, kernel,
    logNoise)`, the reference's argument order; `blockindices` is a list of 0-based index arrays that partition the
    training points.  Lambda is block-diagonal: exact covariance inside each block, the inducing-point approximation
    between blocks.  mll, logdet, alpha and the [noise; mean; kernel] gradient (dmll_noise :328-363, dmll_kern! :274-326) run
    on the GPU (single device)."""
    _mode = 3

    def __init__(self, x, Xu, blockindices, y, mean=None, kernel=None, logNoise=-2.0, device=0, distributed=False):
        if distributed:
            raise ValueError("FSA runs on a single GPU (distributed=True is not supported)")
        x = _as_dxn(x)
        self.blockindices = [np.asarray(b, dtype=np.int64).ravel() for b in blockindices]
        self._block_ptr, self._idx = blocks_to_csr(self.blockindices, x.shape[1])
        self._pending_blocks = True
        super().__init__(x, Xu, y, mean=mean, kernel=kernel, logNoise=logNoise, device=device)

    def append(self, x, y):
        raise ValueError("append is not available for FSA: new observations would need new blocks; build the model again "
                         "with the grown data and blocks")

    def update_mll(self, noise=True, domean=True, kern=True):
        """update_mll! with cK::FullScalePDMat (update_cK! :197-230, `\\` :105-108, logdet :142)."""
        if self._pending_blocks:
            self._eng.set_blocks(self._block_ptr, self._idx)
            self._pending_blocks = False
        return super().update_mll()

    def _cv_prepare(self):
        raise ValueError("cross-validation is not available for FSA")

    def predict_f(self, x, blockindpred, full_cov=False):
        """predict_f(gp, x, blockindpred; full_cov) (:456-477): test block j (0-based index arrays over the columns of x) is
        paired with training block j; test points in no block (or in a block j >= the number of training blocks) get no
        Lambda_xf term.  Without full_cov every point is its own one-point block: the variance is the diagonal of the
        full_cov formula, clamped at 0 (GP.jl:75)."""
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        block_of = test_block_of(blockindpred, x.shape[1])
        xs = np.ascontiguousarray(x.T)
        mu, s2 = self._eng.predict_fsa(xs, block_of, full_cov=full_cov)
        mu = mu + self.mean.mean(xs)
        return (mu, s2) if full_cov else (mu, np.maximum(s2, 0.0))

    def predict_f_grad(self, x, blockindpred=None):
        """predict_f(gp, x, blockindpred) and its gradients with respect to the test inputs, (mu, s2, dmu, ds2) as
        GPE.predict_f_grad: dmu / ds2 are (dim, M), s2 is clamped at 0 (GP.jl:75) and ds2 is 0 where the clamp acts."""
        if blockindpred is None:
            raise ValueError("predict_f_grad: FSA pairs test points with training blocks; pass blockindpred")
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        block_of = test_block_of(blockindpred, x.shape[1])
        xs = np.ascontiguousarray(x.T)
        mu, var, dmu, dvar = self._eng.predict_fsa_grad(xs, block_of, want_var=True)
        mu = mu + self.mean.mean(xs)
        dmu = dmu + self.mean.grad_x(xs)
        dvar[var < 0.0] = 0.0
        return mu, np.maximum(var, 0.0), np.ascontiguousarray(dmu.T), np.ascontiguousarray(dvar.T)

    def predict_y(self, x, blockindpred, full_cov=False):
        mu, s2 = self.predict_f(x, blockindpred, full_cov=full_cov)
        if full_cov:
            return mu, s2 + self.noise_variance() * np.eye(s2.shape[0])
        return mu, s2 + self.noise_variance()

    def rand(self, x, blockindpred, n=1, nugget=1e-10, rng=None):
        """rand(gp, X, n) with the test blocks of predict_f(x, blockindpred; full_cov=true): n posterior draws, (npred, n).
        That covariance is positive semi-definite when every test point is paired with the same training block; over
        several test blocks predictMVN (:413-447) mixes the exact K** with Lambda_xf on the paired blocks only, the matrix
        is in general indefinite and PosDefException is raised, as in the reference."""
        rng = np.random.default_rng() if rng is None else rng
        x = _as_dxn(x)
        if x.shape[0] != self.dim:
            raise ValueError("Gaussian Process object and input observations do not have consistent dimensions")
        block_of = test_block_of(blockindpred, x.shape[1])
        xs = np.ascontiguousarray(x.T)
        z = rng.standard_normal((int(n), xs.shape[0]))
        _, draws = self._eng.rand(xs, z, nugget=nugget, block_of=block_of)
        return (draws + self.mean.mean(xs)[None, :]).T


def test_block_of(blockindpred, npred):
    """0-based test blocks -> block_of[npred] (the training block each test point is paired with, -1 for none);
    ValueError for an index out of range or a test point in two blocks."""
    block_of = np.full(npred, -1, dtype=np.int64)
    for j, ind in enumerate(blockindpred):
        ind = np.asarray(ind, dtype=np.int64).ravel()
        if ind.size and (ind.min() < 0 or ind.max() >= npred):
            raise ValueError("prediction block %d indexes outside the %d test points" % (j, npred))
        if np.any(block_of[ind] != -1) or np.unique(ind).size != ind.size:
            raise ValueError("a test point lies in two prediction blocks")
        block_of[ind] = j
    return block_of
