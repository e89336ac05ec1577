"""Likelihoods of GPA (src/likelihoods/*.jl) -- O(N) host work, like the means: the device computes f = L v + mu and the
gradient through the Cholesky factor, these turn f into log p(y | f) and its derivatives.  Same constructors, parameter
order (log-scale sigma) and formulas as the reference; `predict_obs` is closed-form for Bernoulli and Gaussian and 20-node
Gauss-Hermite quadrature for the rest (likelihoods.jl:16-31)."""
import math

import numpy as np
from scipy.special import gammaln, ndtr

_LOG2PI = math.log(2.0 * math.pi)


def _phi(f):                              # StatsFuns normpdf
    return np.exp(-0.5 * f * f) / math.sqrt(2.0 * math.pi)


class Likelihood:
    def get_params(self):
        return []

    def set_params(self, hyp):
        if len(hyp) != 0:
            raise ValueError("%s has no free parameters" % type(self).__name__)

    def num_params(self):
        return len(self.get_params())

    def check_y(self, y):
        """y as the reference's method signature types it (ValueError == the Julia MethodError for a wrong element type)."""
        y = np.asarray(y)
        if y.ndim != 1 or not (np.issubdtype(y.dtype, np.floating) or np.issubdtype(y.dtype, np.integer)) or y.dtype == bool:
            raise ValueError("%s: y must be a vector of real numbers" % type(self).__name__)
        return y.astype(np.float64)

    def log_dens(self, f, y):
        raise NotImplementedError

    def dlog_dens_df(self, f, y):
        raise NotImplementedError

    def dlog_dens_dtheta(self, f, y):
        """N x num_params matrix (dlog_dens_dθ)"""
        return np.zeros((np.size(f), 0))

    def dlog_dens_dθ(self, f, y):          # the reference's name
        return self.dlog_dens_dtheta(f, y)

    def mean_lik(self, f):
        raise NotImplementedError

    def var_lik(self, f):
        raise NotImplementedError

    def predict_obs(self, fmean, fvar):
        """predictive mean / variance of y from N(fmean, fvar) by 20-node Gauss-Hermite quadrature (likelihoods.jl:16-31)"""
        nodes, weights = np.polynomial.hermite.hermgauss(20)
        weights = weights / math.sqrt(math.pi)
        f = np.asarray(fmean, dtype=np.float64)[:, None] + np.sqrt(2.0 * np.asarray(fvar, dtype=np.float64))[:, None] * nodes[None, :]
        mL = np.column_stack([self.mean_lik(f[:, i]) for i in range(nodes.size)])
        vL = np.column_stack([self.var_lik(f[:, i]) for i in range(nodes.size)])
        mu = mL @ weights
        return mu, (vL + mL ** 2) @ weights - mu ** 2


def _check_counts(lik, y, upper=None):
    y = np.asarray(y)
    if y.ndim != 1 or not np.issubdtype(y.dtype, np.integer) or y.dtype == bool:
        raise ValueError("%s: y must be a vector of integers" % type(lik).__name__)
    if np.any(y < 0) or (upper is not None and np.any(y > upper)):
        raise ValueError("%s: y must lie in 0..%s" % (type(lik).__name__, "n" if upper is not None else "∞"))
    return y.astype(np.int64)


class BernLik(Likelihood):                # bernoulli.jl: theta = Phi(f), y in {false, true}
    def check_y(self, y):
        y = np.asarray(y)
        if y.ndim != 1 or y.dtype != bool:
            raise ValueError("BernLik: y must be a vector of Bool")
        return y.copy()

    def log_dens(self, f, y):             # bernoulli.jl:12-14
        p = ndtr(f)
        return np.where(y, np.log(p), np.log(1.0 - p))

    def dlog_dens_df(self, f, y):         # bernoulli.jl:16-18
        p = ndtr(f)
        return np.where(y, _phi(f) / p, -_phi(f) / (1.0 - p))

    def mean_lik(self, f):
        return ndtr(f)

    def var_lik(self, f):
        p = ndtr(f)
        return p * (1.0 - p)

    def predict_obs(self, fmean, fvar):   # bernoulli.jl:29-32
        p = ndtr(np.asarray(fmean) / np.sqrt(1.0 + np.asarray(fvar)))
        return p, p - p * p


class BinLik(Likelihood):                 # binomial.jl: theta = logistic(f), y in 0..n
    def __init__(self, n):
        if int(n) != n or n < 0:
            raise ValueError("BinLik: the number of trials must be a non-negative integer")
        self.n = int(n)

    def check_y(self, y):
        return _check_counts(self, y, self.n)

    def log_dens(self, f, y):             # binomial.jl:16-19
        th = np.exp(f) / (1.0 + np.exp(f))
        n = self.n
        return gammaln(n + 1.0) - gammaln(y + 1.0) - gammaln(n - y + 1.0) + y * np.log(th) + (n - y) * np.log(1.0 - th)

    def dlog_dens_df(self, f, y):         # binomial.jl:21-23
        return y / (1.0 + np.exp(f)) - (self.n - y) * np.exp(f) / (1.0 + np.exp(f))

    def mean_lik(self, f):
        return self.n * np.exp(f) / (1.0 + np.exp(f))

    def var_lik(self, f):
        return self.n * (np.exp(f) / (1.0 + np.exp(f))) * (1.0 / (1.0 + np.exp(f)))


class ExpLik(Likelihood):                 # exponential.jl: theta = exp(-f)
    def log_dens(self, f, y):             # exponential.jl:13-16
        return -f - np.exp(-f) * y

    def dlog_dens_df(self, f, y):         # exponential.jl:19-21
        return y * np.exp(-f) - 1.0

    def mean_lik(self, f):
        return np.exp(f)

    def var_lik(self, f):
        return np.exp(f) ** 2


class GaussLik(Likelihood):               # gaussian.jl: sigma = exp(lσ)
    def __init__(self, lsigma):
        self.sigma = math.exp(float(lsigma))

    def get_params(self):
        return [math.log(self.sigma)]

    def set_params(self, hyp):
        if len(hyp) != 1:
            raise ValueError("Gaussian/Normal likelihood has only one free parameter")
        self.sigma = math.exp(float(hyp[0]))

    def log_dens(self, f, y):             # gaussian.jl:26-28
        s = self.sigma
        return (-0.5 * _LOG2PI - math.log(s)) - 0.5 * ((y - f) / s) ** 2

    def dlog_dens_df(self, f, y):         # gaussian.jl:31-33
        return (y - f) / self.sigma ** 2

    def dlog_dens_dtheta(self, f, y):     # gaussian.jl:36-38
        s = self.sigma
        return (s * (-1.0 / s + 1.0 / s ** 3 * (y - f) ** 2))[:, None]

    def mean_lik(self, f):
        return np.asarray(f, dtype=np.float64)

    def var_lik(self, f):
        return np.full(np.size(f), self.sigma ** 2)

    def predict_obs(self, fmean, fvar):   # gaussian.jl:55-57
        return np.asarray(fmean), np.asarray(fvar) + self.sigma ** 2


class PoisLik(Likelihood):                # poisson.jl: theta = exp(f)
    def check_y(self, y):
        return _check_counts(self, y)

    def log_dens(self, f, y):             # poisson.jl:13-16
        return y * f - np.exp(f) - gammaln(1.0 + y)

    def dlog_dens_df(self, f, y):         # poisson.jl:19-21
        return y - np.exp(f)

    def mean_lik(self, f):
        return np.exp(f)

    def var_lik(self, f):
        return np.exp(f)


class StuTLik(Likelihood):                # studentT.jl: nu degrees of freedom, scale sigma = exp(lσ)
    def __init__(self, nu, lsigma):
        if int(nu) != nu:
            raise ValueError("StuTLik: the degrees of freedom must be an integer")
        self.nu = int(nu)
        self.sigma = math.exp(float(lsigma))

    def get_params(self):
        return [math.log(self.sigma)]

    def set_params(self, hyp):
        if len(hyp) != 1:
            raise ValueError("Student-t likelihood has only one free parameter")
        self.sigma = math.exp(float(hyp[0]))

    def log_dens(self, f, y):             # studentT.jl:29-34
        nu, s = self.nu, self.sigma
        c = gammaln(0.5 * (nu + 1)) - gammaln(0.5 * nu) - 0.5 * math.log(math.pi * nu) - math.log(s)
        return c - (0.5 * (nu + 1)) * np.log(1.0 + (1.0 / nu) * ((y - f) / s) ** 2)

    def dlog_dens_df(self, f, y):         # studentT.jl:37-41
        nu, s = self.nu, self.sigma
        return (nu + 1) * (y - f) / (nu * s ** 2 + (y - f) ** 2)

    def dlog_dens_dtheta(self, f, y):     # studentT.jl:44-48
        nu, s = self.nu, self.sigma
        return (s * (-1.0 / s + (nu + 1) * (y - f) ** 2 / (nu * s ** 3 + s * (y - f) ** 2)))[:, None]

    def mean_lik(self, f):
        return np.asarray(f, dtype=np.float64)

    def var_lik(self, f):
        return self.sigma ** 2 * (self.nu / (self.nu - 2.0)) * np.ones(np.size(f))
