"""CPU: the host side of the training-input parameters of FITC, DTC, SoR and FSA (gpb200/sparse.py) over a stand-in
FitcEngine backed by the CPU oracles: the [noise; mean; kernel; vec(Xu); vec(X)] order and layout for every combination of
inducing and inputs, one joint engine call per update_dmll, the mean's part added on the host, set_params moving X on the
engine, optimize(inputs=True) rolling back a rejected step, and the distributed rules."""
import numpy as np
import pytest

import gpb200
from gpb200 import capi
import sparse_inputs_grad_oracle as sg
from test_inducing_host_cpu import MODE_NAMES, InducingStub


class InputsStub(InducingStub):
    """InducingStub plus set_inputs / grad_kernel_inputs / comm_init -- TEST ONLY; the device part of dmll/dX is the
    oracle's without the mean's part"""
    reject_x = staticmethod(lambda x: False)

    def set_inputs(self, x_pm):
        self.calls.append("set_inputs")
        self.X = np.array(x_pm)

    def comm_init(self, nranks, rank, uid):
        self.comm = (nranks, rank)

    def factorize(self, theta, ln):
        if self.reject_x(self.X):
            self.rejected += 1
            raise capi.PosDefException(1)
        super().factorize(theta, ln)

    def grad_kernel_inputs(self, want_kernel=True, want_inducing=False):
        self.calls.append("grad_kernel_inputs")
        gk = super().grad_kernel() if want_kernel else None
        gu = super().grad_kernel_inducing(want_kernel=False)[1] if want_inducing else None
        self.calls = [c for c in self.calls if c not in ("grad_kernel", "grad_kernel_inducing")]
        gx = sg.dmll_dx(self.spec, self.X, self.Xu, self.y_minus_mean, self.ln, MODE_NAMES[self.mode], self.blocks)
        return gk, gu, gx


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(capi, "FitcEngine", InputsStub)
    InputsStub.kernel = None
    InputsStub.reject_xu = staticmethod(lambda xu: False)
    InputsStub.reject_x = staticmethod(lambda x: False)


def _model(cls, kernel, n=20, m=3, seed=0, mean=None, **kw):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((2, n))
    y = np.sin(X.sum(axis=0)) + 0.1 * rng.standard_normal(n)
    Xu = rng.standard_normal((2, m))
    InputsStub.kernel = kernel
    mean = gpb200.MeanConst(0.3) if mean is None else mean
    if cls is gpb200.FSA:
        return cls(X, Xu, [np.arange(0, 7), np.arange(7, n)], y, mean, kernel, -1.0, **kw)
    return cls(X, Xu, y, mean, kernel, -1.0, **kw)


COMBOS = [dict(inducing=False, inputs=True), dict(inducing=True, inputs=True)]


@pytest.mark.parametrize("combo", COMBOS)
@pytest.mark.parametrize("cls", [gpb200.FITC, gpb200.DTC, gpb200.SoR, gpb200.FSA])
def test_param_order_and_vec_layout(stub, cls, combo):
    gp = _model(cls, gpb200.SEIso(0.2, 0.1))
    p0 = gp.get_params()
    nu = gp.Xu.size if combo["inducing"] else 0
    p = gp.get_params(**combo)
    assert p.size == p0.size + nu + gp.x.size == gp.num_params(**combo)
    np.testing.assert_array_equal(p[:p0.size], p0)
    if nu:
        np.testing.assert_array_equal(p[p0.size:p0.size + nu], gp.Xu.T.ravel())
    np.testing.assert_array_equal(p[p0.size + nu:], gp.x.T.ravel())              # Julia's vec of the dim x nobs matrix
    np.testing.assert_array_equal(p[p0.size + nu:p0.size + nu + 2], gp.x[:, 0])  # one point after another
    gp.update_target_and_dtarget(**combo)
    assert gp.dtarget.size == p.size
    d_all = gp.dtarget.copy()
    gp.update_target_and_dtarget(inducing=combo["inducing"])
    np.testing.assert_array_equal(d_all[:p0.size + nu], gp.dtarget)             # the prefix is the protocol without X
    gx = gp._eng.grad_kernel_inputs(want_kernel=False)[2] + gp.alpha[:, None] * gp.mean.grad_x(gp._xpm)
    np.testing.assert_array_equal(d_all[p0.size + nu:], gx.ravel())


@pytest.mark.parametrize("combo", COMBOS + [dict(inducing=True, inputs=False), dict(inducing=False, inputs=False)])
def test_set_params_round_trip_every_combination(stub, combo):
    gp = _model(gpb200.FSA, gpb200.SEArd([0.1, -0.2], 0.1))
    p = gp.get_params(**combo)
    q = p + 0.01 * np.arange(p.size)
    gp.set_params(q, **combo)
    np.testing.assert_array_equal(gp.get_params(**combo), q)
    assert ("set_inputs" in gp._eng.calls) == combo["inputs"]
    assert ("set_inducing" in gp._eng.calls) == combo["inducing"]
    if combo["inputs"]:
        np.testing.assert_array_equal(gp._eng.X, gp._xpm)
        np.testing.assert_array_equal(gp.x, gp._xpm.T)
    with pytest.raises(ValueError):
        gp.set_params(q[:-1], **combo)


@pytest.mark.parametrize("flags", [dict(), dict(noise=False, domean=False), dict(kern=False), dict(inducing=True, kern=False)])
def test_one_joint_call_per_update_dmll(stub, flags):
    gp = _model(gpb200.DTC, gpb200.SEArd([0.1, -0.2], 0.1))
    gp._eng.calls.clear()
    gp.update_dmll(inputs=True, **flags)
    assert gp._eng.calls == ["grad_kernel_inputs"]
    assert gp.dmll.size == gp.num_params(inputs=True, **flags)
    gp._eng.calls.clear()
    gp.update_mll_and_dmll(inputs=True, **flags)
    assert gp._eng.calls == ["grad_kernel_inputs"]


def test_mean_part_is_added_on_the_host(stub):
    gp = _model(gpb200.FITC, gpb200.SEIso(0.2, 0.1), mean=gpb200.MeanLin([0.4, -0.7]))
    gp.update_dmll(inputs=True, noise=False, domean=False, kern=False)
    want = sg.dmll_dx(gp.kernel.spec(), gp._xpm, gp.Xu.T, gp.y, -1.0, "FITC", mspec=gp.mean.spec())
    np.testing.assert_allclose(gp.dmll.reshape(-1, 2), want, rtol=1e-12, atol=1e-14)


def test_optimize_inputs_rolls_back_rejected_steps(stub):
    gp = _model(gpb200.FSA, gpb200.SEIso(0.2, 0.1), n=12, m=3)
    x0 = gp.x.copy()
    # a stand-in for a singular FSA block: any training point that moved by more than 0.05 in its first coordinate
    InputsStub.reject_x = staticmethod(lambda x: np.any(np.abs(x[:, 0] - x0[0]) > 0.05))
    m0 = gp.mll
    res = gp.optimize(inputs=True, inducing=True, maxiter=10)
    assert gp._eng.rejected > 0
    assert np.all(np.abs(gp.x[0] - x0[0]) <= 0.05)
    assert np.isfinite(gp.mll) and gp.mll >= m0 - 1e-9
    np.testing.assert_array_equal(gp.get_params(inputs=True, inducing=True), res.x)
    np.testing.assert_array_equal(gp._eng.X, gp._xpm)


def test_distributed_appends_the_slice_and_refuses_optimize_inputs(stub, monkeypatch):
    import os
    import socket
    import torch.distributed as dist
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    monkeypatch.setattr(capi.Engine, "nccl_unique_id", staticmethod(lambda *a: bytes(128)))
    monkeypatch.setitem(os.environ, "MASTER_ADDR", "127.0.0.1")
    monkeypatch.setitem(os.environ, "MASTER_PORT", str(port))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        gp = _model(gpb200.FITC, gpb200.SEIso(0.2, 0.1), distributed=True)
        assert gp._eng.comm == (1, 0)
        gp.update_dmll(inputs=True)
        assert gp.dmll.size == gp.num_params() + gp.x.size
        with pytest.raises(ValueError):
            gp.optimize(inputs=True)
        gp.optimize(maxiter=2)                                     # the other parameters still optimise
    finally:
        dist.destroy_process_group()
