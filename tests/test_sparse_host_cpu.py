"""CPU: the host side of the sparse strategies' parameter protocol and rand (gpb200/sparse.py) over a stand-in FitcEngine
backed by the CPU oracle (the OracleEngine pattern of test_host_cpu.py): [noise; mean; kernel] order, FixedKernel exposure,
set_params / get_params, update_target*, rand's shapes and mean, FSA's test blocks, and optimize's rollback of a rejected
(PosDefException) step."""
import numpy as np
import pytest

import gpb200
from gpb200 import capi
from oracle import gp_oracle as orc
from fsa_oracle import fsa_dmll_kern, fsa_fit

MODES = {0: "FITC", 1: "DTC", 2: "SoR"}


def _unfix(s):
    if s[0] == "Fixed":
        return _unfix(s[1])
    if s[0] in ("Sum", "Prod"):
        return (s[0], _unfix(s[1]), _unfix(s[2]))
    if s[0] == "Masked":
        return ("Masked", _unfix(s[1]), s[2])
    return s


class StubFitcEngine:
    """Stand-in with the FitcEngine interface -- TEST ONLY.  `kernel` is the model's kernel object (set_params changes it in
    place); factorize raises PosDefException when `reject(log_noise)` holds."""
    kernel = None
    reject = staticmethod(lambda ln: False)

    def __init__(self, device=0):
        self.mode, self.blocks, self.rand_calls, self.rejected = 0, None, [], 0

    def set_mode(self, mode):
        self.mode = mode

    def set_data(self, x, xu):
        self.X, self.Xu = np.array(x), np.array(xu)
        self.N, self.d = x.shape

    def set_blocks(self, block_ptr, idx):
        self.blocks = [idx[block_ptr[i]:block_ptr[i + 1]] for i in range(len(block_ptr) - 1)]

    def set_kernel(self, ops, dims, n_theta):
        self.n_theta = n_theta

    def factorize(self, theta, ln):
        if self.reject(ln):
            self.rejected += 1
            raise capi.PosDefException(1)
        self.ln = ln

    def mll(self, r):
        self.spec = _unfix(self.kernel.spec())
        if self.mode == 3:
            self.f = fsa_fit(self.spec, self.X, self.Xu, self.blocks, r, self.ln)
        else:
            self.f = orc.fitc_fit(self.spec, self.X, self.Xu, r, self.ln, mode=MODES[self.mode])
        return self.f["alpha"], self.f["mll"], self.f["logdet"]

    def grad_noise(self):
        return self.f["dmll_noise"]

    def grad_kernel(self):
        if self.mode == 3:
            return fsa_dmll_kern(self.spec, self.X, self.Xu, self.f)
        return orc.fitc_dmll_kern(self.spec, self.X, self.Xu, self.f)

    def rand(self, xs_pm, z, nugget=1e-10, block_of=None):
        if (self.mode == 3) != (block_of is not None):
            raise ValueError("fitc_rand: block_of is required in FSA mode (3) and must be NULL otherwise")
        self.rand_calls.append((xs_pm.copy(), z.copy(), nugget, block_of))
        mu = np.full(xs_pm.shape[0], 5.0)
        return mu, z + mu[None, :]


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(capi, "FitcEngine", StubFitcEngine)
    monkeypatch.setattr(StubFitcEngine, "reject", staticmethod(lambda ln: False))
    return StubFitcEngine


def _data(n=60, m=8, seed=0, noise=0.1):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 2))
    y = np.sin(X.sum(1)) + noise * rng.standard_normal(n)
    return X, X[rng.permutation(n)[:m]], y


def _model(stub, cls, kernel, mean, ln, **kw):
    X, Xu, y = _data(**kw)
    stub.kernel = kernel
    if cls is gpb200.FSA:
        blocks = [np.arange(0, 20), np.arange(20, 45), np.arange(45, X.shape[0])]
        return cls(X.T, Xu.T, blocks, y, mean, kernel, ln), X, Xu, y
    return cls(X.T, Xu.T, y, mean, kernel, ln), X, Xu, y


@pytest.mark.parametrize("cls", [gpb200.FITC, gpb200.DTC, gpb200.SoR, gpb200.FSA])
def test_parameter_order_fixed_kernel_and_lengths(stub, cls):
    k = gpb200.SEIso(0.1, 0.2) + gpb200.fix(gpb200.RQIso(0.3, -0.5, 0.2), "lσ")
    gp, X, Xu, y = _model(stub, cls, k, gpb200.MeanLin([0.1, -0.2]), -1.0)
    assert gp.get_params().tolist() == pytest.approx([-1.0, 0.1, -0.2, 0.1, 0.2, 0.3, 0.2])   # [noise; mean; kernel(free)]
    assert gp.num_params() == 7 and gp.num_params(noise=False) == 6 and gp.num_params(domean=False, kern=False) == 1
    gp.update_target_and_dtarget()
    spec = _unfix(k.spec())
    r = y - X @ np.array([0.1, -0.2])
    if cls is gpb200.FSA:
        o = fsa_fit(spec, X, Xu, gp.blockindices, r, -1.0)
        gk = fsa_dmll_kern(spec, X, Xu, o)
    else:
        o = orc.fitc_fit(spec, X, Xu, r, -1.0, mode=cls.__name__)
        gk = orc.fitc_dmll_kern(spec, X, Xu, o)
    assert gp.target == gp.mll == pytest.approx(o["mll"], rel=1e-12)
    assert gp.dtarget.size == 7
    assert gp.dtarget[0] == pytest.approx(o["dmll_noise"], rel=1e-12)
    assert gp.dtarget[1:3] == pytest.approx(X.T @ o["alpha"], rel=1e-12)        # dmll_mean! of MeanLin
    exposed = gpb200.flatten(k, 2)[3]
    assert exposed == [0, 1, 2, 4] and gp.dtarget[3:] == pytest.approx(gk[exposed], rel=1e-12)
    gp.update_target_and_dtarget(noise=False, domean=False)
    assert gp.dtarget.size == 4
    p = gp.get_params()
    with pytest.raises(ValueError):
        gp.set_params(p[:-1])
    with pytest.raises(ValueError):
        gp.set_params(np.append(p, 0.0))


def test_set_params_get_params_round_trip(stub):
    k = gpb200.SEIso(0.1, 0.2) * gpb200.fix(gpb200.Mat32Iso(0.3, -0.5), "ll")
    gp, X, Xu, y = _model(stub, gpb200.FITC, k, gpb200.MeanConst(0.4), -1.0)
    p = np.array([-0.7, 0.25, 0.15, 0.35, -0.45])
    gp.set_params(p)
    assert np.array_equal(gp.get_params(), p)
    assert gp.logNoise == -0.7 and gp.mean.get_params() == pytest.approx([0.25]) and k.get_params() == pytest.approx([0.15, 0.35, -0.45])
    assert gpb200.flatten(k, 2)[2].tolist() == pytest.approx([0.15, 0.35, 0.3, -0.45])      # the fixed length scale stays
    gp.update_target()
    o = orc.fitc_fit(_unfix(k.spec()), X, Xu, y - 0.25, -0.7)
    assert gp.target == pytest.approx(o["mll"], rel=1e-12)
    gp.set_params([0.5], noise=False, kern=False)                  # mean only
    assert gp.get_params().tolist() == pytest.approx([-0.7, 0.5, 0.15, 0.35, -0.45])
    gp.set_params([-1.5], domean=False, kern=False)                # noise only
    assert gp.logNoise == -1.5


@pytest.mark.parametrize("cls", [gpb200.FITC, gpb200.DTC, gpb200.SoR])
def test_rand_shapes_and_mean(stub, cls):
    gp, X, Xu, y = _model(stub, cls, gpb200.SEIso(0.1, 0.2), gpb200.MeanConst(0.3), -1.0)
    xs = np.random.default_rng(1).standard_normal((2, 11))
    s = gp.rand(xs, n=4, nugget=1e-7, rng=np.random.default_rng(2))
    z = np.random.default_rng(2).standard_normal((4, 11))
    assert s.shape == (11, 4)
    assert np.array_equal(s, (z + 5.0 + 0.3).T)                   # engine draws + mean(x*)
    xp, zz, nugget, block_of = gp._eng.rand_calls[-1]
    assert np.array_equal(xp, xs.T) and np.array_equal(zz, z) and nugget == 1e-7 and block_of is None
    assert gp.rand(xs).shape == (11, 1)
    with pytest.raises(ValueError):
        gp.rand(np.zeros((3, 5)))


def test_fsa_rand_needs_test_blocks(stub):
    gp, X, Xu, y = _model(stub, gpb200.FSA, gpb200.SEIso(0.1, 0.2), gpb200.MeanConst(0.3), -1.0)
    xs = np.random.default_rng(3).standard_normal((2, 9))
    with pytest.raises(TypeError):
        gp.rand(xs)
    with pytest.raises(ValueError, match="two prediction blocks"):
        gp.rand(xs, [[0, 1, 2], [2, 3]])
    with pytest.raises(ValueError):
        gp.rand(xs, [[0, 9]])                                      # index outside the test points
    s = gp.rand(xs, [[4, 0], [], [7]], n=3, rng=np.random.default_rng(4))
    assert s.shape == (9, 3)
    block_of = gp._eng.rand_calls[-1][3]
    assert block_of.tolist() == [0, -1, -1, -1, 0, -1, -1, 2, -1]


def test_optimize_rolls_back_a_rejected_step(stub):
    """Noisy data pull logNoise up; every factorisation above -1.5 raises PosDefException.  optimize rejects those steps
    (optimize.jl:46-87), restores the previous parameters, and ends on an accepted point whose target is consistent."""
    gp, X, Xu, y = _model(stub, gpb200.FITC, gpb200.SEIso(0.1, 0.2), gpb200.MeanZero(), -2.5, noise=1.0)
    stub.reject = staticmethod(lambda ln: ln > -1.5)
    t0 = gp.target
    gp.optimize(domean=False, kern=False, maxiter=30)
    assert gp._eng.rejected >= 1
    assert gp.logNoise <= -1.5 and gp.target > t0
    o = orc.fitc_fit(("SEIso", [0.1, 0.2]), X, Xu, y, gp.logNoise)
    assert gp.target == pytest.approx(o["mll"], rel=1e-12)
    assert gp.kernel.get_params() == pytest.approx([0.1, 0.2])
