"""GPU: the engine handles' device buffers (DevBuf, counted by gpb200_device_bytes).  Every entry point of the dense
engine (one handle and an in-process group of two row-sharded ranks) and of FITC, DTC, SoR and FSA run once and the
engine closed returns the count to its value before creation; a second pass of the same calls on a live engine does not
change it; and a handle taken from mode 0 through FSA blocks back to mode 0 -- which grows
the staging chunk and with it every workspace sized by the chunk -- gives the inverse diagonal and cross-validation
values of a fresh mode-0 engine."""
import numpy as np
import pytest

import gpb200
from gpb200 import capi
import fitc_cv_oracle as fco
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _problem(N, M, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-2.0, 2.0, (M, d))
    return X, y, Xu


def _blocks(N, size, seed):
    idx = np.random.default_rng(seed).permutation(N).astype(np.int64)
    return np.r_[np.arange(0, N, size), N].astype(np.int64), idx


def _setup(eng, mode, X, Xu, y, k, ln, seed=0):
    d = X.shape[1]
    eng.set_mode(mode)
    eng.set_data(np.ascontiguousarray(X), np.ascontiguousarray(Xu))
    ops, dims, theta, _ = gpb200.flatten(k, d)
    eng.set_kernel(ops, dims, theta.size)
    if mode == 3:
        eng.set_blocks(*_blocks(X.shape[0], 150, seed))
    eng.factorize(theta, ln)
    return eng.mll(y)


def _every_call(eng, mode, X, y, Xu, k, ln):
    """one call of every entry point of the sparse handle in `mode` (FSA: mode 3)"""
    rng = np.random.default_rng(7)
    N, d = X.shape
    Ms = 40
    Xs = rng.standard_normal((Ms, d))
    z = rng.standard_normal((3, Ms))
    _setup(eng, mode, X, Xu, y, k, ln)
    eng.grad_noise()
    eng.grad_kernel()
    eng.grad_kernel_inducing()
    eng.grad_kernel_inputs(want_inducing=True)
    if mode == 3:
        block_of = rng.integers(-1, 3, Ms).astype(np.int64)
        eng.predict_fsa(Xs, block_of)
        eng.predict_fsa(Xs, block_of, full_cov=True)
        eng.predict_fsa_grad(Xs, block_of)
        eng.rand(Xs, z, nugget=1e-6, block_of=np.full(Ms, -1, dtype=np.int64))
        eng.set_blocks(*_blocks(N, 200, 1))
    else:
        eng.predict(Xs)
        eng.predict_grad(Xs)
        eng.predict_cov(Xs)
        eng.rand(Xs, z, nugget=1e-6)
        eng.inverse_diag()
        eng.cv_param(0)
        eng.cv_param(-1)
        eng.cv_block(0, np.arange(0, N, 7, dtype=np.int64))
        eng.cv_block(1, np.arange(0, N, 11, dtype=np.int64))
    eng.set_inducing(Xu + 0.01)
    eng.set_inputs(X + 0.01)
    ops, dims, theta, _ = gpb200.flatten(k, d)
    eng.factorize(theta, ln)
    eng.mll(y)


def _dense_calls(eng, X, y, Xs, Xnew, single):
    """GPE / ElasticGPE on `eng`: likelihood, gradients (kernel and inputs), predictions, draws and predictive gradients
    (single handle), CV, append, new data at another N"""
    gp = gpb200.ElasticGPE(X.T, y, gpb200.MeanConst(0.1), gpb200.SEIso(0.2, 0.1), -0.5, engine=eng, capacity=X.shape[0] + 200)
    gp.update_target_and_dtarget(inputs=True)
    gp.predict_f(Xs.T)
    gp.predict_f(Xs.T, full_cov=True)
    if single:
        gp.predict_f_grad(Xs.T)
        gp.rand(Xs.T, n=2, rng=np.random.default_rng(0))
    gp.predict_LOO()
    gp.dlogp_LOO()
    folds = np.array_split(np.arange(X.shape[0]), 5)
    gp.predict_CVfold(folds)
    gp.dlogp_CVfold(folds)
    gp.append(Xnew.T, np.sin(Xnew.sum(1)))
    gp.update_target_and_dtarget()
    gp.fit(X[:500].T, y[:500])                         # a second set_data at another N
    gp.update_target_and_dtarget()
    gp.predict_f(Xs.T)


@pytest.mark.parametrize("group", [False, True])
def test_dense_buffers_are_released_and_do_not_grow(group):
    X, y, _ = _problem(700, 1, 3, 11)
    rng = np.random.default_rng(3)
    Xs, Xnew = rng.standard_normal((33, 3)), rng.standard_normal((60, 3))
    before = capi.device_bytes()
    eng = capi.LocalGroupEngine(2, rb=1) if group else capi.Engine(0)
    try:
        _dense_calls(eng, X, y, Xs, Xnew, not group)
        live = capi.device_bytes()
        assert live > before
        _dense_calls(eng, X, y, Xs, Xnew, not group)    # the same calls again: no per-call growth
        assert capi.device_bytes() == live
    finally:
        eng.close()
    assert capi.device_bytes() == before


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_sparse_buffers_are_released_and_do_not_grow(mode):
    k = gpb200.SEIso(-0.5, 0.1)
    X, y, Xu = _problem(700, 64, 3, mode)
    X2, y2, Xu2 = _problem(1100, 96, 3, mode + 10)
    before = capi.device_bytes()
    eng = capi.FitcEngine(0)
    try:
        _every_call(eng, mode, X, y, Xu, k, -1.0)
        live = capi.device_bytes()
        assert live > before
        _every_call(eng, mode, X, y, Xu, k, -1.0)        # the same calls again: no per-call growth
        assert capi.device_bytes() == live
        _every_call(eng, mode, X2, y2, Xu2, k, -1.0)     # a second set_data at another N and M
    finally:
        eng.close()
    assert capi.device_bytes() == before


def test_mode_switch_remakes_the_cross_validation_workspace():
    k = gpb200.SEIso(-0.6, 0.1)
    N, M, d, ln = 300, 64, 3, -1.0
    X, y, Xu = _problem(N, M, d, 3)
    before = capi.device_bytes()
    sw, ref = capi.FitcEngine(0), capi.FitcEngine(0)
    try:
        _setup(sw, 0, X, Xu, y, k, ln)
        sw.cv_param(0)                                   # cross-validation workspace sized by the small chunk
        ops, dims, theta, _ = gpb200.flatten(k, d)
        sw.set_mode(3)
        sw.set_blocks(*_blocks(N, 150, 0))               # grows the chunk
        sw.factorize(theta, ln)
        sw.mll(y)
        sw.set_mode(0)
        sw.factorize(theta, ln)
        sw.mll(y)
        _setup(ref, 0, X, Xu, y, k, ln)
        Sigma, _ = fco.sigma_and_grads(k.spec(), X, Xu, ln, "FITC")
        w = np.linalg.eigvalsh(orc.cov(k.spec(), Xu) + 1e-10 * np.eye(M))
        ws = np.linalg.eigvalsh(Sigma)
        tol = max(1e-9, 64.0 * float(w[-1] / w[0]) * float(ws[-1] / ws[0]) * EPS)

        def rel(a, b):
            return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))

        assert rel(sw.inverse_diag(), ref.inverse_diag()) <= tol
        for p in (-1, 0, 1):
            za, dg = sw.cv_param(p)
            zr, dr = ref.cv_param(p)
            assert rel(za, zr) <= tol and rel(dg, dr) <= tol, p
    finally:
        sw.close()
        ref.close()
    assert capi.device_bytes() == before
