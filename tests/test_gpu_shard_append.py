"""GPU: ElasticGPE append! on ROW-SHARDED storage (shard_append in csrc/shard_impl.cuh), run as an in-process group of virtual
ranks on one device.  After every append the group is checked against the oracle on the full data, at the tolerances of
test_gpu_shard.py, and against a group GPE built in one batch from the same data."""
import numpy as np
import pytest

from conftest import make_data
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu
RTOL = 1e-10


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def _check_oracle(gp, kern, X, y, ln, Xs, mean):
    o = orc.mll_and_dmll(kern.spec(), X, y, ln, mean.spec())
    assert abs(gp.mll - o["mll"]) <= RTOL * abs(o["mll"]), (gp.mll, o["mll"])
    assert _rel(gp.alpha, o["alpha"]) < RTOL
    mu, s2 = gp.predict_f(Xs.T)
    mo, vo = orc.predict_f(kern.spec(), X, o, Xs, mean.spec())
    assert _rel(mu, mo) < RTOL
    assert np.max(np.abs(s2 - vo)) <= RTOL * np.max(np.abs(vo)) + 1e-13
    gp.update_dmll()
    assert np.allclose(gp.dmll, o["dmll"], rtol=1e-8, atol=1e-10), (gp.dmll, o["dmll"])


# (R, rb, N0, appends): NBp = 128 * rb rows per ownership block
@pytest.mark.parametrize("R,rb,N0,steps", [
    (2, 1, 700, (1,)),                # k = 1
    (4, 4, 1100, (100,)),             # crosses a 128-tile inside one ownership block
    (2, 2, 1500, (100,)),             # crosses into the next ownership block
    (3, 2, 900, (1, 130, 300)),       # three successive appends
    (2, 8, 600, (40,)),               # the old N lies in the first block: everything is refactored
    (5, 1, 1280, (128,)),             # old and new N on tile boundaries
    (8, 1, 1100, (200,)),
    (3, 4, 2000, (64, 1)),
])
def test_group_append_matches_oracle_and_batch(R, rb, N0, steps):
    import gpb200
    Nt = N0 + sum(steps)
    X, y, Xs = make_data(Nt, 3, 300 + R + rb, m=60)
    kern = gpb200.SEIso(0.3, 0.1) if R % 2 == 0 else gpb200.Mat32Iso(0.2, 0.1) + gpb200.RQIso(0.4, -0.3, 0.2)
    mean, ln = gpb200.MeanConst(0.2), -0.5
    eng = gpb200.LocalGroupEngine(R, rb=rb)
    gp = gpb200.ElasticGPE(X[:N0].T, y[:N0], mean, kern, ln, capacity=Nt + 37, engine=eng)
    info0 = [e.storage_info() for e in eng.engines]
    assert all(i["sharded"] and i["rb"] == rb for i in info0), info0
    n = N0
    for k in steps:
        gp.append(X[n:n + k].T, y[n:n + k])
        n += k
        assert gp.nobs == n and eng.N == n and all(e.N == n for e in eng.engines)
        _check_oracle(gp, kern, X[:n], y[:n], ln, Xs, mean)
    assert gp._capacity == Nt + 37                                      # extended in place, never refitted
    assert [e.storage_info() for e in eng.engines] == info0            # append maps no new rows
    # the factor assembled from the ranks' own rows (gp.update_dmll ran the inverse sweep: the factor must be intact)
    Ky = orc.gram(kern.spec(), X, ln)
    U = eng.factor_upper()
    assert np.max(np.abs(U.T @ U - Ky)) <= 1e-11 * np.max(np.abs(Ky))
    rhs = np.cos(X[:, 0])
    assert _rel(eng.solve(rhs), np.linalg.solve(Ky, rhs)) < 1e-9
    assert abs(eng.logdet() - np.linalg.slogdet(Ky)[1]) <= 1e-10 * abs(np.linalg.slogdet(Ky)[1]) + 1e-9
    # a group GPE built in one batch from the same data
    eb = gpb200.LocalGroupEngine(R, rb=rb)
    gb = gpb200.GPE(X.T, y, mean, kern, ln, engine=eb)
    gb.update_target_and_dtarget()
    assert abs(gp.mll - gb.mll) <= RTOL * abs(gb.mll)
    assert _rel(gp.alpha, gb.alpha) < RTOL
    assert np.allclose(gp.dmll, gb.dmll, rtol=1e-8, atol=1e-10)
    mu, s2 = gp.predict_f(Xs.T)
    mb, vb = gb.predict_f(Xs.T)
    assert _rel(mu, mb) < RTOL and np.max(np.abs(s2 - vb)) <= RTOL * np.max(np.abs(vb)) + 1e-13
    eb.close()
    eng.close()


def test_group_append_beyond_capacity_refits():
    import gpb200
    X, y, Xs = make_data(1400, 2, 41, m=30)
    kern = gpb200.Mat52Iso(0.1, 0.2)
    mean = gpb200.MeanZero()
    eng = gpb200.LocalGroupEngine(3, rb=2)
    gp = gpb200.ElasticGPE(X[:1000].T, y[:1000], mean, kern, -0.7, capacity=1050, stepsize=200, engine=eng)
    gp.append(X[1000:1100].T, y[1000:1100])                 # 1100 > 1050: refit with 1300 rows reserved
    assert all(e.storage_info()["sharded"] for e in eng.engines)
    _check_oracle(gp, kern, X[:1100], y[:1100], -0.7, Xs, mean)
    gp.append(X[1100:1300].T, y[1100:1300])                 # in place on the refitted group
    _check_oracle(gp, kern, X[:1300], y[:1300], -0.7, Xs, mean)
    gp.append(X[1300:1400].T, y[1300:1400])                 # 1400 > 1300: refit again
    _check_oracle(gp, kern, X, y, -0.7, Xs, mean)
    eng.close()


def test_group_append_not_positive_definite_then_refit():
    """a duplicate of an old point under the noise kernel at negligible noise gives an exactly zero pivot"""
    import gpb200
    X, y, _ = make_data(400, 2, 47)
    X[350] = X[100]
    kern = gpb200.Noise(0.0)
    eng = gpb200.LocalGroupEngine(3, rb=1)
    gp = gpb200.ElasticGPE(X[:300].T, y[:300], gpb200.MeanZero(), kern, -40.0, capacity=450, engine=eng)
    gp.append(X[300:340].T, y[300:340])
    with pytest.raises(gpb200.PosDefException):
        gp.append(X[340:400].T, y[340:400])
    with pytest.raises(ValueError):                         # the factor is gone until the next factorisation
        eng.solve(np.ones(eng.N))
    gp.logNoise = -0.5
    gp.fit(X.T, y)                                          # the same group refits
    o = orc.fit(kern.spec(), X, y, -0.5)
    assert abs(gp.mll - o["mll"]) <= RTOL * abs(o["mll"])
    assert _rel(gp.alpha, o["alpha"]) < RTOL
    eng.close()


def test_append_error_codes_and_single_gpu_engine():
    import gpb200
    X, y, Xs = make_data(800, 2, 53, m=20)
    kern = gpb200.SEIso(0.1, 0.1)
    eng = gpb200.LocalGroupEngine(2, rb=1)
    gp = gpb200.ElasticGPE(X[:600].T, y[:600], gpb200.MeanZero(), kern, -0.5, capacity=800, engine=eng)
    with pytest.raises(ValueError, match="leader"):
        eng.engines[1].append(X[600:610])                   # collective entry points go through the leader
    gp.append(X[600:700].T, y[600:700])                     # the rejected call left nothing behind
    _check_oracle(gp, kern, X[:700], y[:700], -0.5, Xs, gpb200.MeanZero())
    with pytest.raises(ValueError, match="capacity"):
        eng.append(X[:200])
    # per-point noise needs a refit
    eng.factorize(gp._theta_full(), np.full(700, -0.5))
    with pytest.raises(ValueError, match="scalar logNoise"):
        eng.append(X[700:710])
    eng.close()
    # one GPU: the replicated single-handle append is unchanged
    gs = gpb200.ElasticGPE(X[:600].T, y[:600], gpb200.MeanZero(), kern, -0.5, capacity=800)
    assert not gs._eng.storage_info()["sharded"]
    gs.append(X[600:800].T, y[600:800])
    _check_oracle(gs, kern, X, y, -0.5, Xs, gpb200.MeanZero())
