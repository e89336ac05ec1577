"""CPU: the Full Scale Approximation oracle (tests/fsa_oracle.py) against the dense forms it replaces -- the RNG-free checks
of the reference's test/test_sparse.jl:121-145 -- and the host-side validation of FSA's training blocks."""
import math

import numpy as np
import pytest
import scipy.linalg as sl

from oracle import gp_oracle as orc
from fsa_oracle import fsa_dmll_kern, fsa_fit, fsa_predict_closed, fsa_predict_full, nearest_blocks

SPEC = ("SEIso", [math.log(0.8), math.log(1.3)])


def _data(n=300, seed=3):
    """d = 2; inducing points on a 4 x 4 grid, so that K_uu is well conditioned (cond < 1e3) and the extra 1e-10 nugget of
    Sigma_QR (:227) stays below the 1e-10 relative tolerance"""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 2))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)
    g = np.linspace(-1.5, 1.5, 4)
    Xu = np.array([[a, b] for a in g for b in g])
    return X, y, Xu


def _dense_mll(Sigma, r):
    U = np.linalg.cholesky(Sigma)
    a = sl.cho_solve((U, True), r)
    return -(r @ a + 2 * np.sum(np.log(np.diag(U))) + orc.LOG2PI * r.size) / 2.0, a


def test_fsa_fit_equals_dense_gp_on_sigma():
    X, y, Xu = _data()
    blocks = nearest_blocks(X, Xu)
    o = fsa_fit(SPEC, X, Xu, blocks, y, -1.0, ("MeanConst", 0.1))
    mll, a = _dense_mll(o["Sigma"], o["resid"])                 # GPE on Matrix(cK)  (test_sparse.jl:125-133)
    assert abs(o["mll"] - mll) <= 1e-10 * abs(mll)
    assert abs(o["logdet"] - np.linalg.slogdet(o["Sigma"])[1]) <= 1e-10 * abs(o["logdet"])
    assert np.max(np.abs(o["alpha"] - a)) <= 1e-9 * np.max(np.abs(a))     # cK \ r == Matrix(cK) \ r


def test_fsa_noise_gradient_matches_finite_differences():
    X, y, Xu = _data(n=200, seed=5)
    blocks = nearest_blocks(X, Xu)
    o = fsa_fit(SPEC, X, Xu, blocks, y, -1.0)
    h = 1e-5
    fd = (fsa_fit(SPEC, X, Xu, blocks, y, -1.0 + h)["mll"] - fsa_fit(SPEC, X, Xu, blocks, y, -1.0 - h)["mll"]) / (2 * h)
    assert abs(o["dmll_noise"] - fd) <= 1e-6 * abs(fd)


@pytest.mark.parametrize("spec", [SPEC, ("Sum", ("Mat32Iso", [-0.3, 0.0]), ("RQIso", [-0.5, -0.5, 0.3]))])
def test_fsa_kernel_gradient_matches_finite_differences(spec):
    X, y, Xu = _data(n=160, seed=9)
    blocks = nearest_blocks(X, Xu)
    theta = np.array(_flat(spec))
    o = fsa_fit(spec, X, Xu, blocks, y, -1.0)
    g = fsa_dmll_kern(spec, X, Xu, o)
    h = 1e-5
    for p in range(theta.size):
        tp, tm = theta.copy(), theta.copy()
        tp[p] += h; tm[p] -= h
        fd = (fsa_fit(_unflat(spec, tp), X, Xu, blocks, y, -1.0)["mll"] - fsa_fit(_unflat(spec, tm), X, Xu, blocks, y, -1.0)["mll"]) / (2 * h)
        assert abs(g[p] - fd) <= 1e-6 * max(abs(fd), 1.0), (p, g[p], fd)


def _flat(spec):
    if spec[0] in ("Sum", "Prod"):
        return _flat(spec[1]) + _flat(spec[2])
    return list(spec[1])


def _unflat(spec, theta):
    if spec[0] in ("Sum", "Prod"):
        n = len(_flat(spec[1]))
        return (spec[0], _unflat(spec[1], theta[:n]), _unflat(spec[2], theta[n:]))
    return (spec[0], list(theta))


def test_fsa_predictions_match_predictmvn_and_the_closed_form():
    X, y, Xu = _data(n=300, seed=21)
    blocks = nearest_blocks(X, Xu)
    rng = np.random.default_rng(22)
    Xs = rng.standard_normal((40, 2))
    bpred = nearest_blocks(Xs, Xu)[:10]                        # blocks 10.. of the training set get no test block (zip)
    o = fsa_fit(SPEC, X, Xu, blocks, y, -1.0, ("MeanConst", 0.1))
    mu, S = fsa_predict_full(SPEC, X, Xu, o, Xs, bpred, ("MeanConst", 0.1))
    # predictMVN!(Kxx, cKPD, Qfx + Λfx, mx, alpha) on the dense Matrix(cK)  (test_sparse.jl:77-111)
    from fsa_oracle import _lam_xf
    A = orc.cov(SPEC, Xs, Xu) @ np.linalg.solve(orc.cov(SPEC, Xu) + 1e-10 * np.eye(Xu.shape[0]), orc.cov(SPEC, Xu, X)) \
        + _lam_xf(SPEC, X, Xu, o, Xs, bpred)
    mu_d = 0.1 + A @ o["alpha"]
    S_d = orc.cov(SPEC, Xs, Xs) - A @ np.linalg.solve(o["Sigma"], A.T)
    assert np.max(np.abs(mu - mu_d)) <= 1e-9 * np.max(np.abs(mu_d))
    assert np.max(np.abs(S - S_d)) <= 1e-9 * np.max(np.abs(S_d))
    # the closed form assumes S = K_uu + K_uf Λ⁻¹ K_fu exactly; Σ_QR carries a second 1e-10 nugget (:227), so the two
    # agree to ~1e-10 of the prior scale, not to the last bit
    mc, Sc = fsa_predict_closed(SPEC, X, Xu, o, Xs, bpred, ("MeanConst", 0.1))
    assert np.max(np.abs(mc - mu)) <= 1e-10 * np.max(np.abs(mu))
    assert np.max(np.abs(Sc - S)) <= 1e-9 * np.max(np.abs(S))


def test_test_block_of():
    from gpb200.sparse import test_block_of
    assert test_block_of([np.array([2]), np.array([0, 3])], 5).tolist() == [1, -1, 0, 1, -1]
    with pytest.raises(ValueError):
        test_block_of([np.array([0, 1]), np.array([1])], 3)                # point 1 in two prediction blocks
    with pytest.raises(ValueError):
        test_block_of([np.array([3])], 3)


def test_singleton_blocks_reproduce_fitc():
    X, y, Xu = _data(n=250, seed=7)
    o = fsa_fit(SPEC, X, Xu, [np.array([i]) for i in range(X.shape[0])], y, -1.0)
    f = orc.fitc_fit(SPEC, X, Xu, y, -1.0)
    # FITC's Lambda has no 1e-10 block nugget: the two differ by ~1e-10 tr(Sigma^-1)
    assert abs(o["mll"] - f["mll"]) <= 1e-8 * abs(f["mll"])
    assert np.max(np.abs(o["alpha"] - f["alpha"])) <= 1e-7 * np.max(np.abs(f["alpha"]))
    assert abs(o["dmll_noise"] - f["dmll_noise"]) <= 1e-7 * abs(f["dmll_noise"])
    f["mode"] = "FITC"
    assert np.allclose(fsa_dmll_kern(SPEC, X, Xu, o), orc.fitc_dmll_kern(SPEC, X, Xu, f), rtol=1e-6, atol=1e-7)
    Xs = np.random.default_rng(8).standard_normal((25, 2))
    mu, S = fsa_predict_full(SPEC, X, Xu, o, Xs, [])                      # no test blocks: Λxf = 0
    mf, Sf = orc.fitc_predict_full(SPEC, X, Xu, f, Xs)
    assert np.max(np.abs(mu - mf)) <= 1e-7 * np.max(np.abs(mf))
    assert np.max(np.abs(S - Sf)) <= 1e-7 * np.max(np.abs(Sf))


def test_one_block_is_the_exact_gp():
    X, y, Xu = _data(n=240, seed=11)
    o = fsa_fit(SPEC, X, Xu, [np.arange(X.shape[0])], y, -1.0, ("MeanConst", 0.1))
    e = orc.mll_and_dmll(SPEC, X, y, -1.0, ("MeanConst", 0.1), extra_nugget=1e-10)
    assert abs(o["mll"] - e["mll"]) <= 1e-9 * abs(e["mll"])
    assert np.max(np.abs(o["alpha"] - e["alpha"])) <= 1e-8 * np.max(np.abs(e["alpha"]))
    assert abs(o["dmll_noise"] - e["dmll"][0]) <= 1e-7 * abs(e["dmll"][0])
    assert np.allclose(fsa_dmll_kern(SPEC, X, Xu, o), e["dmll_kernel"], rtol=1e-6, atol=1e-7)
    Xs = np.random.default_rng(12).standard_normal((30, 2))
    mu, S = fsa_predict_full(SPEC, X, Xu, o, Xs, [np.arange(30)], ("MeanConst", 0.1))
    mo, So = orc.predict_f(SPEC, X, e, Xs, ("MeanConst", 0.1), full_cov=True)
    assert np.max(np.abs(mu - mo)) <= 1e-8 * np.max(np.abs(mo))
    assert np.max(np.abs(S - So)) <= 1e-8 * np.max(np.abs(So))


def test_blocks_to_csr_and_validation():
    from gpb200.sparse import blocks_to_csr
    bp, idx = blocks_to_csr([np.array([2, 0]), np.array([], dtype=int), np.array([1, 3])], 4)
    assert bp.tolist() == [0, 2, 2, 4] and idx.tolist() == [2, 0, 1, 3]
    with pytest.raises(ValueError):
        blocks_to_csr([np.array([0, 1]), np.array([1, 2])], 3)           # 1 twice, not a partition
    with pytest.raises(ValueError):
        blocks_to_csr([np.array([0, 1])], 3)                             # 2 missing
    with pytest.raises(ValueError):
        blocks_to_csr([np.array([0, 5])], 2)                             # out of range
    with pytest.raises(ValueError):
        blocks_to_csr([np.arange(2049), np.arange(2049, 2050)], 2050)    # block over 2048 points
    bp, idx = blocks_to_csr([np.arange(2048), np.arange(2048, 2050)], 2050)
    assert bp.tolist() == [0, 2048, 2050]


def test_fsa_rejects_bad_blocks_and_distributed_before_touching_the_device():
    import gpb200 as g
    X, y, Xu = _data(n=20)
    with pytest.raises(ValueError):
        g.FSA(X.T, Xu.T, [np.arange(10), np.arange(9, 20)], y, g.MeanZero(), g.SEIso(0.0, 0.0), -1.0)
    with pytest.raises(ValueError):
        g.FSA(X.T, Xu.T, [np.arange(20)], y, g.MeanZero(), g.SEIso(0.0, 0.0), -1.0, distributed=True)


def test_header_declares_set_blocks_as_bound():
    import gpb200.capi as capi
    assert "gpb200_fitc_set_blocks" in capi.declared_symbols()


def test_julia_shim_binds_the_fsa_entry_points_like_the_header():
    """B200FSA's update_cK! and predict_f reach gpb200_fitc_set_blocks / _predict_fsa with the header's argument types"""
    from test_julia_shim import C2JL, JL, _ctype, header_prototypes, julia_ccalls
    protos = header_prototypes()
    calls = {c[0]: c for c in julia_ccalls()}
    for name in ("gpb200_fitc_set_blocks", "gpb200_fitc_predict_fsa"):
        assert name in calls and name in protos, name
        _, _, tlist, values = calls[name]
        assert len(tlist) == len(protos[name]) == len(values), name
        for jt, cdecl in zip(tlist, protos[name]):
            assert jt in C2JL[_ctype(cdecl)], (name, jt, cdecl)
    src = open(JL).read()
    assert "struct B200FSA" in src and "Int64[i - 1 for b in cs.blockindices for i in b]" in src      # 1-based -> 0-based
    assert "block_of[i] = j - 1" in src
