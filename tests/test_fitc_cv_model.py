"""CPU: cross-validation for the sparse strategies without forming the N x N inverse.

* the numpy model of the device schedule (tests/fitc_cv_model.py: chunks smaller than N, two streaming passes) against the
  dense inverse of Sigma for FITC, DTC and SoR;
* the dense dSigma_j of tests/fitc_cv_oracle.py against central differences of Sigma;
* the refit identity: the LOO / fold predictions read off Sigma^-1 equal predict_y of the model refitted without the held-out
  points (FITC and SoR, whose predictive covariance is their training covariance; DTC's is not);
* the FITC host assembly over a stub engine, against the oracle's literal cross-validation bodies;
* the Julia shim binds the three new entry points with the header's signatures."""
import math
import os
import re

import numpy as np
import pytest

import fitc_cv_oracle as fco
from fitc_cv_model import SparseCV
from oracle import gp_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPECS = {"SEIso": ("SEIso", [-0.6, 0.1]),
         "Mat32+Noise": ("Sum", ("Mat32Iso", [-0.4, -0.1]), ("Noise", [-1.3]))}


def _problem(N, M, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-2.0, 2.0, (M, d))
    return X, y, Xu


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


@pytest.mark.parametrize("kname", sorted(SPECS))
@pytest.mark.parametrize("strategy", ["FITC", "DTC", "SoR"])
@pytest.mark.parametrize("N,M,chunk", [(300, 20, 128), (1100, 45, 256)])
def test_chunked_schedule_matches_dense_inverse(strategy, kname, N, M, chunk):
    spec = SPECS[kname]
    mode = "FITC" if strategy == "FITC" else "SoR"                    # DTC trains with SoR's covariance
    X, y, Xu = _problem(N, M, 2, N + M)
    model = SparseCV(spec, X, Xu, -1.0, mode, chunk=chunk)
    Sigma, grads = fco.sigma_and_grads(spec, X, Xu, -1.0, mode)
    invS = np.linalg.inv(Sigma)
    alpha = invS @ y
    assert _rel(model.inverse_diag(), np.diag(invS)) < 1e-8
    V = np.sort(np.random.default_rng(0).choice(N, 37, replace=False))
    assert _rel(model.cv_block(0, V), invS[np.ix_(V, V)]) < 1e-8
    for p in [-1] + list(range(len(grads))):
        dS = np.eye(N) if p < 0 else grads[p]
        za, dg = model.cv_param(p, alpha)
        zo, do = fco.cv_vectors(invS, dS, alpha)
        M_j = invS @ dS @ invS
        assert _rel(za, zo) < 1e-7 and _rel(dg, do) < 1e-7, (p, _rel(za, zo), _rel(dg, do))
        assert _rel(model.cv_block(1, V), M_j[np.ix_(V, V)]) < 1e-7


@pytest.mark.parametrize("mode", ["FITC", "SoR"])
def test_dense_dsigma_matches_central_differences(mode):
    X, _, Xu = _problem(60, 12, 2, 3)
    spec = SPECS["Mat32+Noise"]
    _, grads = fco.sigma_and_grads(spec, X, Xu, -1.0, mode)
    theta = [-0.4, -0.1, -1.3]
    h = 1e-6
    for p in range(len(theta)):
        def sig(t):
            s = ("Sum", ("Mat32Iso", t[:2]), ("Noise", t[2:]))
            return fco.sigma_and_grads(s, X, Xu, -1.0, mode)[0]
        tp, tm = list(theta), list(theta)
        tp[p] += h; tm[p] -= h
        fd = (sig(tp) - sig(tm)) / (2 * h)
        assert _rel(grads[p], fd) < 1e-6, (p, _rel(grads[p], fd))


@pytest.mark.parametrize("mode", ["FITC", "SoR"])
def test_refit_identity(mode):
    """LOO mean / variance of point i = predict_y at x_i of the model refitted without i; a fold likewise (full covariance)"""
    spec = SPECS["SEIso"]
    N, M = 120, 15
    X, y, Xu = _problem(N, M, 2, 8)
    ln = -1.0
    Sigma, _ = fco.sigma_and_grads(spec, X, Xu, ln, mode)
    f = fco.cv_dict(Sigma, np.linalg.solve(Sigma, y))
    mu, s2 = orc.predict_loo(f, y)
    nv = math.exp(2 * ln)
    for i in (0, 17, 119):
        keep = np.delete(np.arange(N), i)
        o = orc.fitc_fit(spec, X[keep], Xu, y[keep], ln, mode=mode)
        m_i, v_i = orc.fitc_predict(spec, X[keep], Xu, o, X[i:i + 1])
        assert abs(mu[i] - m_i[0]) <= 1e-7 * max(1.0, abs(m_i[0])) and abs(s2[i] - (v_i[0] + nv)) <= 1e-7 * (v_i[0] + nv)
    V = np.array([3, 40, 41, 99])
    mus, Ss = orc.predict_cvfold(f, y, [V])
    keep = np.setdiff1d(np.arange(N), V)
    o = orc.fitc_fit(spec, X[keep], Xu, y[keep], ln, mode=mode)
    mo, So = orc.fitc_predict_full(spec, X[keep], Xu, o, X[V])
    So = So + nv * np.eye(V.size)
    assert _rel(mus[0], mo) < 1e-7
    if mode == "SoR":
        assert _rel(Ss[0], So) < 1e-7
    else:   # FITC's predictive covariance keeps K_** - Q_** off the diagonal, its training prior only Lambda's diagonal
        assert _rel(np.diag(Ss[0]), np.diag(So)) < 1e-7


class _StubEngine:
    """the three FitcEngine CV calls from a dense Sigma (host assembly test)"""

    def __init__(self, Sigma, grads):
        self.invS, self.grads, self._Mj = np.linalg.inv(Sigma), grads, None

    def inverse_diag(self):
        return np.diag(self.invS).copy()

    def cv_param(self, param, alpha=None):
        dS = np.eye(self.invS.shape[0]) if param < 0 else self.grads[param]
        self._Mj = self.invS @ dS @ self.invS
        return fco.cv_vectors(self.invS, dS, self._alpha)

    def cv_block(self, which, idx):
        src = self.invS if which == 0 else self._Mj
        return src[np.ix_(idx, idx)]


@pytest.mark.parametrize("strategy", ["FITC", "SoR", "FSA"])
def test_host_assembly_over_stub_engine(strategy):
    import gpb200 as g
    spec = SPECS["Mat32+Noise"]
    mode = "FITC" if strategy == "FITC" else "SoR"
    N = 150
    X, y, Xu = _problem(N, 14, 2, 21)
    ln = -0.8
    Sigma, grads = fco.sigma_and_grads(spec, X, Xu, ln, mode)
    alpha = np.linalg.solve(Sigma, y)
    gp = object.__new__(getattr(g, strategy))
    gp.y, gp.alpha, gp.logNoise, gp.mean, gp._exposed = y, alpha, ln, g.MeanZero(), np.arange(len(grads))
    gp._eng = _StubEngine(Sigma, grads)
    gp._eng._alpha = alpha
    folds = np.array_split(np.random.default_rng(4).permutation(N), 5)
    if strategy == "FSA":
        for call in (gp.predict_LOO, gp.dlogp_LOO, lambda: gp.logp_CVfold(folds), lambda: gp.dlogp_CVfold(folds)):
            with pytest.raises(ValueError):
                call()
        return
    f = fco.cv_dict(Sigma, alpha)
    mu, s2 = gp.predict_LOO()
    mo, so = orc.predict_loo(f, y)
    assert _rel(mu, mo) < 1e-10 and _rel(s2, so) < 1e-10
    assert abs(gp.logp_LOO() - orc.logp_loo(f, y)) < 1e-10 * abs(orc.logp_loo(f, y))
    assert _rel(gp.dlogp_LOO(), fco.dlogp_loo(Sigma, grads, alpha, y, ln)) < 1e-9
    assert abs(gp.logp_CVfold(folds) - orc.logp_cvfold(f, y, folds)) < 1e-9 * abs(orc.logp_cvfold(f, y, folds))
    assert _rel(gp.dlogp_CVfold(folds), fco.dlogp_cvfold(Sigma, grads, alpha, y, ln, folds)) < 1e-9
    assert gp.dlogp_LOO(noise=False).size == len(grads) and gp.dlogp_CVfold(folds, kern=False).size == 1


def _header_signature(name):
    with open(os.path.join(ROOT, "include", "gpb200.h")) as fh:
        src = fh.read()
    m = re.search(r"int\s+%s\(([^)]*)\)" % name, src)
    assert m, name
    return [a.strip().rsplit(" ", 1)[0].replace(" *", "*").replace("const ", "") for a in m.group(1).split(",")]


def test_julia_shim_binds_the_sparse_cv_entry_points():
    with open(os.path.join(ROOT, "gaussianprocesses.jl_b200", "julia", "GPB200.jl")) as fh:
        jl = fh.read()
    julia_of = {"gpb200_fitc*": "Ptr{Cvoid}", "double*": "Ptr{Float64}", "int64_t*": "Ptr{Int64}", "int32_t": "Int32",
                "int64_t": "Int64"}
    for name in ("gpb200_fitc_get_inverse_diag", "gpb200_fitc_cv_param", "gpb200_fitc_cv_block"):
        want = [julia_of[t] for t in _header_signature(name)]
        m = re.search(r":%s\s*,\s*LIB\)\s*,\s*Cint\s*,\s*\(([^)]*)\)" % name, jl)
        assert m, "%s is not ccall'ed" % name
        got = [t.strip() for t in m.group(1).split(",") if t.strip()]
        assert got == want, (name, got, want)
