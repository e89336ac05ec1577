"""CPU: the host side of the inducing-point parameters (gpb200/sparse.py) over a stand-in FitcEngine backed by the CPU oracles:
the [noise; mean; kernel; vec(Xu)] order and layout, inducing=False identical to the protocol without it, one joint engine
call per update_dmll(inducing=True), set_params moving Xu on the engine, and optimize(inducing=True) rolling back a
rejected (PosDefException) step."""
import numpy as np
import pytest

import gpb200
from gpb200 import capi
import inducing_grad_oracle as ig
from test_sparse_host_cpu import MODES, StubFitcEngine

MODE_NAMES = {**MODES, 3: "FSA"}


class InducingStub(StubFitcEngine):
    """StubFitcEngine plus set_inducing / grad_kernel_inducing -- TEST ONLY; counts the gradient calls"""
    reject_xu = staticmethod(lambda xu: False)

    def __init__(self, device=0):
        super().__init__(device)
        self.calls = []

    def set_inducing(self, xu_pm):
        self.calls.append("set_inducing")
        self.Xu = np.array(xu_pm)

    def factorize(self, theta, ln):
        if self.reject_xu(self.Xu):
            self.rejected += 1
            raise capi.PosDefException(1)
        super().factorize(theta, ln)

    def grad_kernel(self):
        self.calls.append("grad_kernel")
        return super().grad_kernel()

    def grad_kernel_inducing(self, want_kernel=True):
        self.calls.append("grad_kernel_inducing")
        gk = super().grad_kernel() if want_kernel else None
        gx = ig.dmll_dxu(self.spec, self.X, self.Xu, self.y_minus_mean, self.ln, MODE_NAMES[self.mode], self.blocks)
        return gk, gx

    def mll(self, r):
        self.y_minus_mean = np.array(r)
        return super().mll(r)


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(capi, "FitcEngine", InducingStub)
    InducingStub.kernel = None
    InducingStub.reject_xu = staticmethod(lambda xu: False)


def _model(cls, kernel, n=30, m=4, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((2, n))
    y = np.sin(X.sum(axis=0)) + 0.1 * rng.standard_normal(n)
    Xu = rng.standard_normal((2, m))
    InducingStub.kernel = kernel
    if cls is gpb200.FSA:
        return cls(X, Xu, [np.arange(0, 11), np.arange(11, n)], y, gpb200.MeanConst(0.3), kernel, -1.0)
    return cls(X, Xu, y, gpb200.MeanConst(0.3), kernel, -1.0)


@pytest.mark.parametrize("cls", [gpb200.FITC, gpb200.DTC, gpb200.SoR, gpb200.FSA])
def test_param_order_and_vec_layout(stub, cls):
    gp = _model(cls, gpb200.SEIso(0.2, 0.1))
    p0 = gp.get_params()
    p = gp.get_params(inducing=True)
    assert p.size == p0.size + gp.Xu.size == gp.num_params(inducing=True)
    np.testing.assert_array_equal(p[:p0.size], p0)
    np.testing.assert_array_equal(p[p0.size:], gp.Xu.T.ravel())          # Julia's vec of the dim x M matrix
    np.testing.assert_array_equal(p[p0.size:p0.size + 2], gp.Xu[:, 0])   # one point after another
    gp.update_target_and_dtarget(inducing=True)
    assert gp.dtarget.size == p.size
    gk = gp._eng.grad_kernel_inducing()[1]
    np.testing.assert_array_equal(gp.dtarget[p0.size:], gk.ravel())
    # kernel part is grad_kernel's: the same [noise; mean; kernel] prefix as without inducing
    d_inc = gp.dtarget.copy()
    gp.update_target_and_dtarget()
    np.testing.assert_array_equal(gp.dtarget, d_inc[:p0.size])


@pytest.mark.parametrize("cls", [gpb200.FITC, gpb200.FSA])
def test_inducing_false_is_unchanged(stub, cls):
    gp = _model(cls, gpb200.SEIso(0.2, 0.1) + gpb200.fix(gpb200.RQIso(0.1, 0.0, 0.2), "l"))
    p = gp.get_params()
    assert gp.get_params(inducing=False).tolist() == p.tolist() == gpb200.GPE.get_params(gp).tolist()
    assert gp.num_params() == gp.num_params(inducing=False) == p.size
    gp.update_dmll()
    a = gp.dmll.copy()
    gp.update_dmll(inducing=False)
    np.testing.assert_array_equal(gp.dmll, a)
    assert "grad_kernel_inducing" not in gp._eng.calls and "set_inducing" not in gp._eng.calls
    gp.set_params(p + 0.01)
    np.testing.assert_array_equal(gp.get_params(), p + 0.01)
    assert "set_inducing" not in gp._eng.calls


@pytest.mark.parametrize("flags", [dict(), dict(noise=False, domean=False), dict(kern=False), dict(noise=False, kern=False)])
def test_one_joint_call_per_update_dmll(stub, flags):
    gp = _model(gpb200.FITC, gpb200.SEArd([0.1, -0.2], 0.1))
    gp._eng.calls.clear()
    gp.update_dmll(inducing=True, **flags)
    assert gp._eng.calls == ["grad_kernel_inducing"]
    n = gp.num_params(inducing=True, **flags)
    assert gp.dmll.size == n
    gp._eng.calls.clear()
    gp.update_mll_and_dmll(inducing=True, **flags)
    assert gp._eng.calls == ["grad_kernel_inducing"]


def test_set_params_moves_xu(stub):
    gp = _model(gpb200.SoR, gpb200.SEIso(0.2, 0.1))
    p = gp.get_params(inducing=True)
    q = p.copy()
    q[-gp.Xu.size:] += np.arange(gp.Xu.size) * 0.01
    gp.set_params(q, inducing=True)
    assert gp._eng.calls[-1] == "set_inducing"
    np.testing.assert_array_equal(gp.Xu.T.ravel(), q[-gp.Xu.size:])
    np.testing.assert_array_equal(gp._eng.Xu, gp.Xu.T)
    np.testing.assert_array_equal(gp.get_params(inducing=True), q)
    with pytest.raises(ValueError):
        gp.set_params(q[:-1], inducing=True)


def test_optimize_inducing_rolls_back_rejected_steps(stub):
    gp = _model(gpb200.FITC, gpb200.SEIso(0.2, 0.1), n=25, m=3)
    x0 = gp.Xu.copy()
    # a stand-in for two inducing points meeting: any point that moved by more than 0.05 in its first coordinate
    InducingStub.reject_xu = staticmethod(lambda xu: np.any(np.abs(xu[:, 0] - x0[0]) > 0.05))
    m0 = gp.mll
    res = gp.optimize(inducing=True, maxiter=15)
    assert gp._eng.rejected > 0
    assert np.all(np.abs(gp.Xu[0] - x0[0]) <= 0.05)
    assert np.isfinite(gp.mll) and gp.mll >= m0 - 1e-9
    np.testing.assert_array_equal(gp.get_params(inducing=True), res.x)
