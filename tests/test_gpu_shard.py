"""GPU: the ROW-SHARDED storage + schedules (csrc/shard_impl.cuh; config C4's layout) on ONE device, as an in-process group
of virtual ranks (gpb200_group_create): every rank maps only its own block rows of the N x N factor / inverse (CUDA VMM), so
a stray read of another rank's rows faults; collectives are event-ordered copies.  Checked against the CPU oracle at the
tolerances of the single-GPU parity tests, and bit-for-bit independence from the rank count is NOT required (different
summation orders) -- agreement with the oracle is."""
import numpy as np
import pytest

from conftest import make_data
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu
RTOL = 1e-10


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def _group_gp(R, rb, X, y, kern, mean, ln):
    import gpb200
    eng = gpb200.LocalGroupEngine(R, rb=rb)
    return gpb200.GPE(X.T, y, mean, kern, ln, engine=eng), eng


@pytest.mark.parametrize("R,rb,N", [(2, 1, 700), (2, 4, 1500), (3, 2, 1500), (3, 4, 1700), (4, 1, 1100), (4, 2, 2300),
                                    (5, 1, 1300), (8, 1, 2100), (2, 8, 2500), (8, 2, 4200)])
def test_sharded_group_matches_oracle(R, rb, N):
    import gpb200
    d = 3
    X, y, Xs = make_data(N, d, 100 + R + rb, m=130)
    kern = gpb200.SEIso(0.3, 0.1) if (R + rb) % 2 == 0 else gpb200.Mat32Iso(0.2, 0.1) + gpb200.RQIso(0.4, -0.3, 0.2)
    gp, eng = _group_gp(R, rb, X, y, kern, gpb200.MeanConst(0.2), -0.5)
    info = [e.storage_info() for e in eng.engines]
    assert all(i["sharded"] and i["nranks"] == R and i["rb"] == rb and i["tma"] for i in info), info
    gp.update_target_and_dtarget()
    o = orc.mll_and_dmll(kern.spec(), X, y, -0.5, ("MeanConst", 0.2))
    assert abs(gp.mll - o["mll"]) <= RTOL * abs(o["mll"])
    assert _rel(gp.alpha, o["alpha"]) < RTOL
    assert np.allclose(gp.dmll, o["dmll"], rtol=1e-8, atol=1e-10), (gp.dmll, o["dmll"])
    # factor and inverse assembled from the ranks' own rows
    U = eng.factor_upper()
    Ky = orc.gram(kern.spec(), X, -0.5)
    assert np.max(np.abs(U.T @ U - Ky)) <= 1e-11 * np.max(np.abs(Ky))
    Kinv = eng.inverse()
    assert np.max(np.abs(Kinv @ Ky - np.eye(N))) <= 1e-8
    # solve(), logdet
    rhs = np.cos(X[:, 0])
    assert _rel(eng.solve(rhs), np.linalg.solve(Ky, rhs)) < 1e-9
    assert abs(eng.logdet() - np.linalg.slogdet(Ky)[1]) <= 1e-10 * abs(np.linalg.slogdet(Ky)[1]) + 1e-9
    # predictions (mean, variance, full covariance)
    mu, s2 = gp.predict_f(Xs.T)
    mo, vo = orc.predict_f(kern.spec(), X, o, Xs, ("MeanConst", 0.2))
    assert _rel(mu, mo) < RTOL
    assert np.max(np.abs(s2 - vo)) <= RTOL * np.max(np.abs(vo)) + 1e-13
    mu2, cov = gp.predict_f(Xs.T[:, :40], full_cov=True)
    _, co = orc.predict_f(kern.spec(), X, o, Xs[:40], ("MeanConst", 0.2), full_cov=True)
    assert np.max(np.abs(cov - co)) <= 1e-9 * np.max(np.abs(co)) + 1e-12
    # further evaluations with new hyper-parameters reuse the storage (and must not race with the previous schedules)
    gp.set_params(gp.get_params() + 0.02)
    gp.update_target_and_dtarget()
    gp.set_params(gp.get_params() + 0.03)
    gp.update_target_and_dtarget()
    k2 = kern.spec()
    o2 = orc.mll_and_dmll(k2, X, y, gp.logNoise, gp.mean.spec())
    assert abs(gp.mll - o2["mll"]) <= RTOL * abs(o2["mll"])
    assert np.allclose(gp.dmll, o2["dmll"], rtol=1e-8, atol=1e-10)
    eng.close()


def test_sharded_storage_is_physically_sparse():
    """N = 8192: a 128-row tile is 8 MB = 4 allocation pages, so each of the 4 ranks backs exactly a quarter of F and G
    (test/memory.jl:14-19 counterpart: 2 N x N buffers over R devices instead of 4 on one host)."""
    import gpb200
    N, d, R = 8192, 4, 4
    X, y, Xs = make_data(N, d, 9, m=64)
    kern = gpb200.SEIso(0.4, 0.2)
    gp, eng = _group_gp(R, 2, X, y, kern, gpb200.MeanZero(), -0.3)
    full = 8 * N * N
    for e in eng.engines:
        i = e.storage_info()
        assert i["sharded"] and i["bytes_F"] == full // R and i["bytes_G"] == full // R, i
    gp.update_target_and_dtarget()
    # size-independent checks (the oracle needs ~minutes here): residual of alpha on sampled rows, trace identity, FD
    rows = np.random.default_rng(0).choice(N, 32, replace=False)
    Kr = orc.cov(kern.spec(), X[rows], X)
    Kr[np.arange(32), rows] += np.exp(-0.6)
    assert np.max(np.abs(Kr @ gp.alpha - y[rows])) <= 1e-10 * np.max(np.abs(y))
    p0 = gp.get_params(); g0 = gp.dtarget.copy()
    dirv = np.array([0.3, -0.5, 0.4]); h = 1e-4
    gp.set_params(p0 + h * dirv); gp.update_target(); tp = gp.target
    gp.set_params(p0 - h * dirv); gp.update_target(); tm = gp.target
    assert abs((tp - tm) / (2 * h) - g0 @ dirv) <= 1e-6 * abs(g0 @ dirv) + 1e-6
    gp.set_params(p0); gp.update_target()
    mu, s2 = gp.predict_f(Xs.T)
    mu_tr, _ = gp.predict_f(X[rows].T)
    assert np.max(np.abs(mu_tr - orc.cov(kern.spec(), X[rows], X) @ gp.alpha)) <= 1e-10 * np.max(np.abs(mu_tr)) + 1e-12
    assert np.all(s2 >= 0) and np.all(s2 <= np.exp(0.4) * (1 + 1e-12))
    eng.close()


def test_sharded_not_positive_definite_is_reported_and_recoverable():
    import gpb200
    X, y, _ = make_data(900, 2, 3)
    X[500] = X[100]                                  # duplicate point + no noise: singular Gram matrix
    kern = gpb200.SEIso(0.0, 0.0)
    eng = gpb200.LocalGroupEngine(3, rb=2)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), kern, -0.5, engine=eng)
    with pytest.raises(gpb200.PosDefException):
        eng.factorize(np.array([0.0, 0.0]), -40.0)
    gp.update_target()                               # same handles, new hyper-parameters: works again
    o = orc.fit(kern.spec(), X, y, -0.5)
    assert abs(gp.mll - o["mll"]) <= RTOL * abs(o["mll"])
    eng.close()


def test_group_requires_leader_and_matching_state():
    import gpb200
    eng = gpb200.LocalGroupEngine(2)
    X, y, _ = make_data(300, 2, 1)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), gpb200.SEIso(0.1, 0.1), -0.5, engine=eng)
    with pytest.raises(ValueError):
        eng.engines[1].factorize(np.array([0.1, 0.1]), -0.5)        # collective calls go through the leader
    eng.close()
