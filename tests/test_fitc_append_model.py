"""CPU: a numpy model of the update equations of gpb200_fitc_append (csrc/fitc_engine.cu) against the dense restatement of
the sparse covariance (tests/fitc_cv_oracle.py, `sigma_and_grads`) on the concatenated data.  The model keeps only what the
device keeps -- Sigma_QR, b = K_uf Lambda^-1 r, s = r'Lambda^-1 r, l = sum log Lambda_i and N -- and adds each batch of new
rows to them:
    Sigma_QR += K_un Lambda_n^-1 K_nu,  b += K_un Lambda_n^-1 r_n,  s += sum r_n^2 / Lambda_n,  l += sum log Lambda_n
    u = Sigma_QR^-1 b,  mll = -1/2 (s - b'u + logdet Sigma_QR - logdet K_uu + l + N log 2 pi)
Lambda_n: sigma^2 + k_ii - |L_uu^-1 k_ui|^2 (FITC) or sigma^2 (DTC, SoR).  The first state is built the way factorize + mll
build it, then rebuilt as L_s L_s' as the first device append does.  Against the dense Sigma the model starts Sigma_QR from
K_uu + 1e-10 I, the K_uu of Q, so that the two differ by rounding only; the engine adds make_posdef!'s second 1e-10."""
import math

import numpy as np
import pytest

import fitc_cv_oracle as fco
from oracle import gp_oracle as orc


class AppendModel:
    def __init__(self, spec, Xu, log_noise, mode, s_nugget=1e-10):
        self.spec, self.Xu, self.mode = spec, np.asarray(Xu, dtype=np.float64), mode
        m = self.Xu.shape[0]
        self.s2 = math.exp(2.0 * log_noise)
        self.Kuu = orc.cov(spec, self.Xu) + 1e-10 * np.eye(m)             # eu: K_uu + 1e-10 I
        self.Luu = np.linalg.cholesky(self.Kuu)
        self.S = orc.cov(spec, self.Xu) + s_nugget * np.eye(m)            # es: K_uu + 2e-10 I on the device
        self.b = np.zeros(m)
        self.s = self.l = 0.0
        self.n = 0

    def lam(self, X):
        if self.mode != "FITC":
            return np.full(X.shape[0], self.s2)
        V = np.linalg.solve(self.Luu, orc.cov(self.spec, self.Xu, X))
        return self.s2 + orc._kdiag(self.spec, X) - np.sum(V * V, axis=0)

    def add(self, X, r):
        X = np.asarray(X, dtype=np.float64)
        lam = self.lam(X)
        Kun = orc.cov(self.spec, self.Xu, X)
        self.S = self.S + (Kun / lam) @ Kun.T
        self.b = self.b + Kun @ (r / lam)
        self.s += float(np.sum(r * r / lam))
        self.l += float(np.sum(np.log(lam)))
        self.n += X.shape[0]

    def rebuild(self):
        """Sigma_QR as L_s L_s' (what the first append after a factorize starts from)"""
        L = np.linalg.cholesky(self.S)
        self.S = L @ L.T

    def state(self):
        u = np.linalg.solve(self.S, self.b)
        ld = np.linalg.slogdet(self.S)[1] - np.linalg.slogdet(self.Kuu)[1] + self.l
        mll = -0.5 * (self.s - self.b @ u + ld + self.n * math.log(2.0 * math.pi))
        return mll, ld, u


def _dense(spec, X, Xu, r, log_noise, mode):
    """mll and logdet of the dense Sigma on the concatenated data; u from its definition Sigma_QR^-1 K_uf Lambda^-1 r"""
    Sigma, _ = fco.sigma_and_grads(spec, X, Xu, log_noise, "FITC" if mode == "FITC" else "SoR")
    ld = np.linalg.slogdet(Sigma)[1]
    mll = -0.5 * (r @ np.linalg.solve(Sigma, r) + ld + X.shape[0] * math.log(2.0 * math.pi))
    model = AppendModel(spec, Xu, log_noise, mode)
    model.add(X, r)
    return mll, ld, np.linalg.solve(model.S, model.b)


def _problem(n, m, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    r = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)
    Xu = rng.uniform(-2.0, 2.0, (m, d))
    return X, r, Xu


SPECS = {"SEIso": ("SEIso", [-0.4, 0.1]),
         "Mat32+RQ": ("Sum", ("Mat32Iso", [-0.3, -0.1]), ("RQIso", [0.2, -0.2, 0.3]))}


@pytest.mark.parametrize("k", [1, 5, 40])
@pytest.mark.parametrize("kname", sorted(SPECS))
@pytest.mark.parametrize("mode", ["FITC", "DTC", "SoR"])
def test_update_equations_match_the_concatenated_data(mode, kname, k):
    spec = SPECS[kname]
    n0, m, d, ln = 120, 20, 2, -1.2
    X, r, Xu = _problem(n0 + k, m, d, 7 * k + len(kname))
    model = AppendModel(spec, Xu, ln, mode)
    model.add(X[:n0], r[:n0])
    model.rebuild()
    model.add(X[n0:], r[n0:])
    mll, ld, u = model.state()
    mo, lo, uo = _dense(spec, X, Xu, r, ln, mode)
    assert abs(mll - mo) <= 1e-9 * abs(mo), (mll, mo)
    assert abs(ld - lo) <= 1e-9 * abs(lo), (ld, lo)
    assert np.max(np.abs(u - uo)) <= 1e-8 * np.max(np.abs(uo))


@pytest.mark.parametrize("mode", ["FITC", "DTC", "SoR"])
def test_chained_appends(mode):
    spec = SPECS["Mat32+RQ"]
    m, d, ln = 16, 3, -1.0
    sizes = [50, 1, 7, 1, 30, 3, 12]
    X, r, Xu = _problem(sum(sizes), m, d, 11)
    model = AppendModel(spec, Xu, ln, mode)
    edges = np.cumsum([0] + sizes)
    model.add(X[:edges[1]], r[:edges[1]])
    model.rebuild()
    for a, b in zip(edges[1:-1], edges[2:]):
        model.add(X[a:b], r[a:b])
        mll, ld, u = model.state()
        mo, lo, uo = _dense(spec, X[:b], Xu, r[:b], ln, mode)
        assert abs(mll - mo) <= 1e-9 * abs(mo) and abs(ld - lo) <= 1e-9 * abs(lo)
        assert np.max(np.abs(u - uo)) <= 1e-8 * np.max(np.abs(uo))


def test_model_matches_the_oracle_fit():
    """the model's state from scratch is the mll and logdet of the oracle's fitc_fit (the engine's reference)"""
    spec = SPECS["SEIso"]
    X, r, Xu = _problem(90, 12, 2, 3)
    for mode in ("FITC", "SoR"):
        model = AppendModel(spec, Xu, -1.1, mode, s_nugget=2e-10)
        model.add(X, r)
        mll, ld, _ = model.state()
        o = orc.fitc_fit(spec, X, Xu, r, -1.1, mode=mode)
        assert mll == pytest.approx(o["mll"], rel=1e-9) and ld == pytest.approx(o["logdet"], rel=1e-9)
