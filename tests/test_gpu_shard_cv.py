"""GPU: cross-validation on ROW-SHARDED storage (shard_cv_* in csrc/shard_impl.cuh), run as in-process groups of virtual ranks on
one device.  LOO and k-fold values and gradients against the oracle (at the tolerances of
test_gpu_parity.py::test_crossvalidation_on_device_matches_oracle) and against a single-GPU engine on the same inputs; the
distributed pieces themselves (exactly symmetric blocks, a bitwise inverse diagonal, reproducible cv_param); state rules;
physically sparse work matrices; launch counts."""
import json

import numpy as np
import pytest

from conftest import make_data
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def _kernel(i):
    import gpb200 as g
    if i == 0:                                                   # the kernel of the single-GPU CV parity test
        return g.Mat52Iso(0.3, 0.1) + g.fix(g.SEIso(-0.2, 0.3), "lσ")
    return g.Mat32Iso(0.2, 0.1) + g.RQIso(0.4, -0.3, 0.2)


def _folds(N, nbp, seed):
    """a contiguous fold straddling the first ownership-block boundary, a scattered one, and one across the last tile"""
    rng = np.random.default_rng(seed)
    f0 = np.arange(nbp - 60, nbp + 70)
    rest = np.setdiff1d(np.arange(N), f0)
    f1 = np.sort(rng.choice(rest, 150, replace=False))
    f2 = np.setdiff1d(np.arange(N - 200, N), np.concatenate([f0, f1]))
    return [f0, f1, f2]


@pytest.mark.parametrize("R,rb,N,kern", [
    (2, 1, 700, 0),
    (3, 2, 1500, 1),
    (4, 1, 1100, 0),
    (8, 1, 2100, 1),
    (2, 4, 2500, 0),
    (5, 1, 1280, 1),                  # N on a tile boundary
])
def test_group_cv_matches_oracle_and_single_gpu(R, rb, N, kern):
    import gpb200
    X, y, _ = make_data(N, 2, 600 + R * 10 + rb)
    k = _kernel(kern)
    ln = -0.7
    eng = gpb200.LocalGroupEngine(R, rb=rb)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), k, ln, engine=eng)
    gp.update_target_and_dtarget()
    assert all(e.storage_info()["sharded"] and e.storage_info()["rb"] == rb for e in eng.engines)
    Kinv0 = eng.inverse()
    one = gpb200.GPE(X.T, y, gpb200.MeanZero(), k, ln)              # single GPU, same inputs
    one.update_target_and_dtarget()
    f = orc.fit(k.spec(), X, y, ln)
    folds = _folds(N, 128 * rb, N)

    mu, s2 = gp.predict_LOO()
    mo, so = orc.predict_loo(f, y)
    assert _rel(mu, mo) < 1e-9 and _rel(s2, so) < 1e-9
    m1, v1 = one.predict_LOO()
    assert _rel(mu, m1) < 1e-9 and _rel(s2, v1) < 1e-9
    lo = orc.logp_loo(f, y)
    assert abs(gp.logp_LOO() - lo) <= 1e-9 * abs(lo)
    g = gp.dlogp_LOO(noise=True, kern=True)
    go = orc.dlogp_loo(k.spec(), X, y, f, ln)
    assert g.shape == go.shape and np.allclose(g, go, rtol=1e-7, atol=1e-9), (g, go)
    assert np.allclose(g, one.dlogp_LOO(noise=True, kern=True), rtol=1e-7, atol=1e-9)

    mus, Sigs = gp.predict_CVfold(folds)
    muo, Sigo = orc.predict_cvfold(f, y, folds)
    mu1, Sig1 = one.predict_CVfold(folds)
    for a, b, c, dd, a1, c1 in zip(mus, muo, Sigs, Sigo, mu1, Sig1):
        assert _rel(a, b) < 1e-8 and _rel(c, dd) < 1e-8
        assert _rel(a, a1) < 1e-8 and _rel(c, c1) < 1e-8
    lf = orc.logp_cvfold(f, y, folds)
    assert abs(gp.logp_CVfold(folds) - lf) <= 1e-8 * abs(lf)
    gf = gp.dlogp_CVfold(folds, noise=True, kern=True)
    gfo = orc.dlogp_cvfold(k.spec(), X, y, f, ln, folds)
    assert np.allclose(gf, gfo, rtol=1e-6, atol=1e-8), (gf, gfo)
    assert np.allclose(gf, one.dlogp_CVfold(folds, noise=True, kern=True), rtol=1e-6, atol=1e-8)

    # the distributed pieces: exactly symmetric blocks, close to the single-GPU blocks
    j = int(gp._exposed[0])
    za, dz = eng.cv_param(j)
    za1, dz1 = one._eng.cv_param(j)
    assert _rel(za, za1) < 1e-8 and _rel(dz, dz1) < 1e-8
    for V in folds:
        B0, B1 = eng.cv_block(0, V), eng.cv_block(1, V)
        assert np.array_equal(B0, B0.T) and np.array_equal(B1, B1.T)
        assert _rel(B0, one._eng.cv_block(0, V)) < 1e-9
        assert _rel(B1, one._eng.cv_block(1, V)) < 1e-8
    zb, db = eng.cv_param(j)                                        # fixed reduction order: bitwise repeatable
    assert np.array_equal(za, zb) and np.array_equal(dz, db)
    assert np.array_equal(B1, eng.cv_block(1, folds[-1]))
    zn, dn = eng.cv_param(-1)
    zn2, dn2 = eng.cv_param(-1)
    assert np.array_equal(zn, zn2) and np.array_equal(dn, dn2)
    assert _rel(zn, one._eng.cv_param(-1)[0]) < 1e-8

    # the inverse diagonal is read from the ranks' own rows: bitwise the diagonal of the host-assembled inverse
    assert np.array_equal(eng.inverse_diag(), np.diag(eng.inverse()))
    # CV left the lower triangle of K^-1 alone: the inverse and the trace gradient are unchanged
    assert np.array_equal(eng.inverse(), Kinv0)
    gp.update_dmll()
    o = orc.mll_and_dmll(k.spec(), X, y, ln)
    assert np.allclose(gp.dmll, o["dmll"], rtol=1e-8, atol=1e-10)
    eng.close()


def test_group_cv_state_and_errors():
    import gpb200
    X, y, _ = make_data(700, 2, 71)
    k = _kernel(1)
    ln = -0.6
    eng = gpb200.LocalGroupEngine(2, rb=1)
    gp = gpb200.GPE(X[:600].T, y[:600], gpb200.MeanZero(), k, ln, capacity=700, engine=eng)
    V = np.arange(100, 300)
    # before grad_prepare
    for call in (lambda: eng.cv_param(0), lambda: eng.cv_block(0, V), eng.inverse_diag):
        with pytest.raises(ValueError, match="grad_prepare"):
            call()
    eng.grad_prepare()
    with pytest.raises(ValueError, match="cv_param first"):
        eng.cv_block(1, V)
    # collective entry points go through the leader
    for call in (lambda: eng.engines[1].cv_param(0), lambda: eng.engines[1].cv_block(0, V), eng.engines[1].inverse_diag):
        with pytest.raises(ValueError, match="leader"):
            call()
    with pytest.raises(ValueError, match="out of range"):
        eng.cv_block(0, [0, 600])
    a0 = eng.cv_param(0)
    B1 = eng.cv_block(1, V)
    # a refactorisation drops K^-1 and M_j
    gp.update_mll()
    for call in (lambda: eng.cv_param(0), lambda: eng.cv_block(1, V)):
        with pytest.raises(ValueError, match="grad_prepare"):
            call()
    eng.grad_prepare()
    with pytest.raises(ValueError, match="cv_param first"):
        eng.cv_block(1, V)
    a1 = eng.cv_param(0)                                            # same hyper-parameters: the same numbers
    assert np.array_equal(a0[0], a1[0]) and np.array_equal(a0[1], a1[1]) and np.array_equal(B1, eng.cv_block(1, V))
    # append extends the factor in place and drops the inverse; CV then runs on the 700 points
    gp.append(X[600:].T, y[600:])
    assert eng.N == 700
    for call in (lambda: eng.cv_param(0), lambda: eng.cv_block(1, V)):
        with pytest.raises(ValueError, match="grad_prepare"):
            call()
    f = orc.fit(k.spec(), X, y, ln)
    mu, s2 = gp.predict_LOO()
    mo, so = orc.predict_loo(f, y)
    assert _rel(mu, mo) < 1e-9 and _rel(s2, so) < 1e-9
    g = gp.dlogp_LOO()
    go = orc.dlogp_loo(k.spec(), X, y, f, ln)
    assert np.allclose(g, go, rtol=1e-7, atol=1e-9), (g, go)
    eng.close()
    # one GPU: the CV work buffers are counted once they exist
    e1 = gpb200.GPE(X.T, y, gpb200.MeanZero(), k, ln)
    e1._eng.grad_prepare()
    assert e1._eng.storage_info()["bytes_cv"] == 0
    e1._eng.cv_param(0)
    assert e1._eng.storage_info()["bytes_cv"] == 2 * 8 * 768 * 768


def test_group_cv_work_matrices_are_physically_sparse():
    import gpb200
    N, R = 8192, 4
    X, y, _ = make_data(N, 2, 73)
    eng = gpb200.LocalGroupEngine(R)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), gpb200.SEIso(0.3, 0.1), -0.5, engine=eng)
    gp.update_target_and_dtarget()
    assert [e.storage_info()["bytes_cv"] for e in eng.engines] == [0] * R
    za, dz = eng.cv_param(0)
    assert [e.storage_info()["bytes_cv"] for e in eng.engines] == [2 * 8 * N * N // R] * R
    assert np.all(np.isfinite(za)) and np.all(np.isfinite(dz))
    eng.close()


def _device_kernels(fn, tmp_path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "launches.pt.trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    return sum(1 for e in events if e.get("cat") == "kernel" and not e.get("name", "").startswith(("Memcpy", "Memset")))


def test_group_cv_launch_count(tmp_path):
    """The profiler can miss kernel records (on an H100 it has reported fewer kernels than were launched, repeatably for a
    given call, in this test and in tests/test_gpu_launch_count.py), but it never reports a kernel that did not run: every
    kernel it records must have been counted.  Up to three identical attempts per step; the table is printed."""
    import gpb200
    X, y, _ = make_data(1500, 3, 75)
    eng = gpb200.LocalGroupEngine(2, rb=1)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), _kernel(1), -0.5, engine=eng)
    gp.update_target_and_dtarget()
    V = np.arange(50, 400)

    def fresh_inverse():                                            # the next cv_param symmetrises K^-1 again
        gp.update_mll()
        eng.grad_prepare()
    steps = [
        ("cv_param(j)+sym", fresh_inverse, lambda: eng.cv_param(1)),
        ("cv_param(j)", None, lambda: eng.cv_param(0)),
        ("cv_param(-1)", None, lambda: eng.cv_param(-1)),
        ("cv_block", None, lambda: (eng.cv_block(0, V), eng.cv_block(1, V))),
        ("inverse_diag", None, eng.inverse_diag),
    ]
    for name, prep, fn in steps:
        tries = []
        for _ in range(3):
            if prep:
                prep()
            c0 = eng.launch_count()
            kernels = _device_kernels(fn, tmp_path)
            tries.append((eng.launch_count() - c0, kernels))
            if tries[-1][0] == kernels:
                break
        print("launch count 2 ranks %-16s (counted, device): %s" % (name, tries))
        assert all(k <= c for c, k in tries), (name, tries)
    eng.close()


@pytest.mark.slow
def test_group_loo_gradient_finite_difference_16k():
    """N = 16384 on 4 ranks: the directional finite difference of logp_LOO matches dlogp_LOO"""
    import gpb200
    N = 16384
    X, y, _ = make_data(N, 3, 77)
    eng = gpb200.LocalGroupEngine(4)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), gpb200.Mat32Iso(0.2, 0.1), -0.5, engine=eng)
    p0 = gp.get_params(noise=True, domean=False, kern=True)
    g = gp.dlogp_LOO(noise=True, kern=True)
    v = np.array([0.6, -0.5, 0.62])
    h = 1e-4

    def at(p):
        gp.set_params(p, noise=True, domean=False, kern=True)
        gp.update_target()
        return gp.logp_LOO()
    fd = (at(p0 + h * v) - at(p0 - h * v)) / (2 * h)
    assert abs(fd - g @ v) <= 1e-5 * max(abs(fd), 1.0), (fd, g @ v)
    eng.close()
