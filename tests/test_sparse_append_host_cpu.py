"""CPU: the host side of append for the sparse strategies (gpb200/sparse.py) over a stand-in FitcEngine backed by the CPU
oracle (the pattern of tests/test_sparse_host_cpu.py): append forwards r = y - m(x) of the new rows only, sets mll / target
and the data, leaves alpha None until a gradient or cross-validation call refreshes it through update_mll, FSA refuses, and
a distributed model passes only its own slice."""
import numpy as np
import pytest

import gpb200
from gpb200 import capi
from oracle import gp_oracle as orc

MODES = {0: "FITC", 1: "DTC", 2: "SoR"}


class StubFitcEngine:
    """Stand-in with the FitcEngine interface -- TEST ONLY.  append records its arguments and returns the oracle's mll of
    the grown data; `kernel` is the model's kernel object."""
    kernel = None

    def __init__(self, device=0):
        self.mode, self.appends, self.factorizations, self.comm = 0, [], 0, None

    def comm_init(self, nranks, rank, uid):
        self.comm = (nranks, rank)

    def set_mode(self, mode):
        self.mode = mode

    def set_data(self, x, xu):
        self.X, self.Xu = np.array(x), np.array(xu)
        self.N, self.d = x.shape

    def set_blocks(self, block_ptr, idx):
        pass

    def set_kernel(self, ops, dims, n_theta):
        self.n_theta = n_theta

    def factorize(self, theta, ln):
        self.ln = ln
        self.factorizations += 1

    def _fit(self, r):
        return orc.fitc_fit(self.kernel.spec(), self.X, self.Xu, r, self.ln, mode=MODES.get(self.mode, "FITC"))

    def mll(self, r):
        if r.shape != (self.N,):
            raise ValueError("fitc_mll: y must have length N")
        self.r = np.array(r)
        self.f = self._fit(self.r)
        return self.f["alpha"], self.f["mll"], self.f["logdet"]

    def append(self, xnew_pm, r_new):
        self.appends.append((np.array(xnew_pm), np.array(r_new)))
        self.X = np.concatenate([self.X, xnew_pm])
        self.r = np.concatenate([self.r, r_new])
        self.N = self.X.shape[0]
        self.f = None                                            # alpha is not available until mll
        f = self._fit(self.r)
        return f["mll"], f["logdet"]

    def grad_noise(self):
        if self.f is None:
            raise ValueError("fitc_grad_noise: factorize and mll first")
        return self.f["dmll_noise"]

    def grad_kernel(self):
        if self.f is None:
            raise ValueError("fitc_grad_kernel: factorize and mll first")
        return orc.fitc_dmll_kern(self.kernel.spec(), self.X, self.Xu, self.f)

    def inverse_diag(self):
        if self.f is None:
            raise ValueError("fitc_get_inverse_diag: factorize and mll first")
        return np.ones(self.N)


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(capi, "FitcEngine", StubFitcEngine)
    return StubFitcEngine


def _data(n=70, m=8, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 2))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)
    return X, X[rng.permutation(n)[:m]], y


@pytest.mark.parametrize("cls", [gpb200.FITC, gpb200.DTC, gpb200.SoR])
def test_append_forwards_residuals_and_refreshes_alpha_lazily(stub, cls):
    X, Xu, y = _data()
    k = gpb200.SEIso(0.1, 0.2)
    stub.kernel = k
    mean = gpb200.MeanLin([0.3, -0.2])
    gp = cls(X[:50].T, Xu.T, y[:50], mean, k, -1.0)
    assert gp._eng.factorizations == 1
    gp.append(X[50:].T, y[50:])
    xa, ra = gp._eng.appends[-1]
    assert np.array_equal(xa, X[50:]) and np.allclose(ra, y[50:] - X[50:] @ np.array([0.3, -0.2]), rtol=0, atol=1e-15)
    o = orc.fitc_fit(k.spec(), X, Xu, y - X @ np.array([0.3, -0.2]), -1.0, mode=cls.__name__)
    assert gp.mll == pytest.approx(o["mll"], rel=1e-12) and gp.target == gp.mll and gp.logdet == pytest.approx(o["logdet"], rel=1e-12)
    assert gp.alpha is None and gp.nobs == 70 and gp.x.shape == (2, 70) and gp.y.size == 70
    assert np.array_equal(gp._xpm, X) and gp._eng.factorizations == 1
    gp.update_dmll()                                             # alpha first: update_mll refits on the grown data
    assert gp._eng.factorizations == 2 and gp.alpha is not None
    assert np.allclose(gp.alpha, o["alpha"], rtol=1e-12, atol=1e-14)
    assert gp.dmll[0] == pytest.approx(o["dmll_noise"], rel=1e-12)
    gp.append(X[:3].T, y[:3])                                    # a second append; CV also refreshes alpha first
    gp._cv_prepare()
    assert gp._eng.factorizations == 3 and gp.alpha.size == 73
    gp.append(X[:1].T, y[0])                                     # one observation, a scalar target
    assert gp.nobs == 74 and gp._eng.appends[-1][0].shape == (1, 2)


def test_append_argument_checks(stub):
    X, Xu, y = _data()
    stub.kernel = gpb200.SEIso(0.0, 0.0)
    gp = gpb200.FITC(X[:50].T, Xu.T, y[:50], gpb200.MeanZero(), stub.kernel, -1.0)
    with pytest.raises(ValueError, match="observations, but"):
        gp.append(X[50:].T, y[50:55])
    with pytest.raises(ValueError, match="same dimension"):
        gp.append(np.zeros((3, 4)), np.zeros(4))
    assert gp._eng.appends == [] and gp.nobs == 50


def test_fsa_append_raises(stub):
    X, Xu, y = _data()
    stub.kernel = gpb200.SEIso(0.0, 0.0)
    gp = gpb200.FSA(X[:50].T, Xu.T, [np.arange(25), np.arange(25, 50)], y[:50], gpb200.MeanZero(), stub.kernel, -1.0)
    with pytest.raises(ValueError, match="FSA"):
        gp.append(X[50:].T, y[50:])


def test_distributed_model_appends_its_slice(stub, monkeypatch):
    import torch.distributed as dist
    import gpb200.dist as gd
    monkeypatch.setattr(dist, "get_rank", lambda *a, **k: 1)
    monkeypatch.setattr(dist, "get_world_size", lambda *a, **k: 2)
    monkeypatch.setattr(gd, "broadcast_bytes", lambda b, src=0: b"\0" * 128)
    monkeypatch.setattr(capi.Engine, "nccl_unique_id", staticmethod(lambda *a: b"\0" * 128), raising=False)
    X, Xu, y = _data()
    stub.kernel = gpb200.SEIso(0.0, 0.0)
    lo, hi = 35, 50                                              # this rank's initial and new rows
    gp = gpb200.FITC(X[lo:hi].T, Xu.T, y[lo:hi], gpb200.MeanZero(), stub.kernel, -1.0, distributed=True)
    assert gp._eng.comm == (2, 1)
    gp.append(X[60:70].T, y[60:70])
    xa, ra = gp._eng.appends[-1]
    assert np.array_equal(xa, X[60:70]) and np.array_equal(ra, y[60:70]) and gp.nobs == 25
    gp.append(np.zeros((2, 0)), np.zeros(0))                     # a rank may append nothing in a collective step
    assert gp._eng.appends[-1][0].shape == (0, 2) and gp.nobs == 25
