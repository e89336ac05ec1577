"""CPU: the FSA restatement of the predictive gradients (fsa_xgrad_oracle.fsa_predict_f_grad) against fsa_oracle's closed
form, the literal predictMVN and its central differences; the host side of FSA.predict_f_grad with a stub engine; and
the Julia shim's Dual method for B200FSA, checked statically against the header."""
import os
import re

import numpy as np
import pytest

import gpb200 as g
from conftest import kernel_zoo, make_data
from fsa_oracle import fsa_fit, fsa_predict_closed, fsa_predict_full, nearest_blocks
from oracle import gp_oracle as orc
import xgrad_oracle as xo
from fsa_xgrad_oracle import fsa_predict_f_grad

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(spec, seed=3):
    """N = 90, d = 3, 9 inducing points, nearest-inducing-point blocks; 14 test points: paired ones (one equal to a
    training input of its own block), unpaired ones and one in a test block past the last training block"""
    X, y, Xs = make_data(90, 3, seed, m=12)
    Xu = X[::10].copy()
    blocks = nearest_blocks(X, Xu)
    f = fsa_fit(spec, X, Xu, blocks, y, -1.0, ("MeanLin", [0.3, -0.2, 0.1]))
    b0 = next(j for j, b in enumerate(f["blocks"]) if b.size >= 2)
    Xs = np.vstack([Xs, X[f["blocks"][b0][1]][None, :], Xs[0:1] + 0.05])
    bpred = [[] for _ in range(len(blocks) + 1)]
    bpred[b0] = [0, 1, 2, 12]
    nb = next(j for j, b in enumerate(f["blocks"]) if b.size and j != b0)
    bpred[nb] = [3, 4]
    bpred[len(blocks)] = [13]                                   # past the last training block: no Lambda_xf term
    return X, Xu, Xs, f, bpred                                 # 5 .. 11 unpaired


def _block_of(bpred, n):
    return g.sparse.test_block_of(bpred, n)


@pytest.mark.parametrize("name", ["SEIso", "Mat32Ard", "SE*RQ", "Poly"])
def test_fsa_xgrad_oracle(name):
    spec = dict(kernel_zoo(3))[name].spec()
    mspec = ("MeanLin", [0.3, -0.2, 0.1])
    X, Xu, Xs, f, bpred = _case(spec)
    mu, var, dmu, dvar = fsa_predict_f_grad(spec, X, Xu, f, Xs, bpred, mspec)
    mc, Sc = fsa_predict_closed(spec, X, Xu, f, Xs, bpred, mspec)
    mf, Sf = fsa_predict_full(spec, X, Xu, f, Xs, bpred, mspec)
    np.testing.assert_allclose(mu, mc, rtol=0, atol=1e-12 * np.max(np.abs(mc)))
    np.testing.assert_allclose(var, np.diag(Sc), rtol=0, atol=1e-12 * np.max(np.abs(np.diag(Sc))) + 1e-14)
    # the literal predictMVN solves with Sigma_QR's second 1e-10 nugget (:227), which the closed form leaves out, as
    # test_fsa_cpu states: the gap measured here is ~1e-12 cond(K_uu) of the prior scale (2e-10 for SEIso, 2e-8 for Poly
    # with cond(K_uu) = 3e4)
    tol = max(1e-9, 4e-12 * np.linalg.cond(f["Uuu"]) ** 2)
    np.testing.assert_allclose(mu, mf, rtol=0, atol=tol * np.max(np.abs(mf)))
    np.testing.assert_allclose(var, np.diag(Sf), rtol=0, atol=tol * np.max(np.abs(np.diag(Sf))))
    if name == "Poly":
        assert np.max(np.abs(xo.kdiag_dx(spec, Xs))) > 0.1          # the non-stationary D_** term is exercised
    # central differences of the literal predictMVN, one test point at a time (var = the diagonal of its covariance)
    h = 1e-5
    for p in range(3):
        E = np.zeros_like(Xs); E[:, p] = h
        mp, Sp = fsa_predict_full(spec, X, Xu, f, Xs + E, bpred, mspec)
        mm, Sm = fsa_predict_full(spec, X, Xu, f, Xs - E, bpred, mspec)
        fd_mu, fd_var = (mp - mm) / (2 * h), (np.diag(Sp) - np.diag(Sm)) / (2 * h)
        assert np.max(np.abs(dmu[:, p] - fd_mu)) <= 1e-6 * max(np.max(np.abs(dmu)), 1.0), name
        assert np.max(np.abs(dvar[:, p] - fd_var)) <= 1e-6 * max(np.max(np.abs(dvar)), 1e-3), name


def test_fsa_xgrad_unpaired_is_fitc():
    """with no test point paired, c = 0 and the formula is FITC's on FSA's fit (u, K_uu, Sigma_QR)"""
    spec = dict(kernel_zoo(3))["Mat32Ard"].spec()
    X, Xu, Xs, f, _ = _case(spec)
    mspec = ("MeanZero",)
    mu, var, dmu, dvar = fsa_predict_f_grad(spec, X, Xu, f, Xs, [], mspec)
    mo, vo, dmo, dvo = xo.fitc_predict_f_grad(spec, X, Xu, f, Xs, mspec)
    for a, b in ((mu, mo), (var, vo), (dmu, dmo), (dvar, dvo)):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12 * max(np.max(np.abs(b)), 1.0))


class _StubFsaEngine:
    def __init__(self, var):
        self.var = np.asarray(var, dtype=np.float64)
        self.block_of = None

    def predict_fsa_grad(self, xs, block_of, want_var=True):
        self.block_of = np.asarray(block_of).copy()
        M, d = xs.shape
        dmu = np.arange(M * d, dtype=np.float64).reshape(M, d)
        return np.ones(M), self.var.copy(), dmu, -dmu - 1.0


def test_fsa_predict_f_grad_host():
    """(dim, M) layout, the mean's gradient, GP.jl:75's clamp (ds2 = 0 where var < 0) and the test blocks passed down"""
    gp = g.FSA.__new__(g.FSA)
    gp.dim, gp.mean = 2, g.MeanLin([0.5, -2.0])
    gp._eng = _StubFsaEngine([0.3, -1e-12, 0.0])
    xs = np.array([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]])
    mu, s2, dmu, ds2 = gp.predict_f_grad(xs.T, [[2], [], [0]])
    np.testing.assert_array_equal(gp._eng.block_of, [2, -1, 0])
    np.testing.assert_array_equal(mu, 1.0 + xs @ np.array([0.5, -2.0]))
    np.testing.assert_array_equal(s2, [0.3, 0.0, 0.0])
    assert dmu.shape == (2, 3) and ds2.shape == (2, 3)
    np.testing.assert_array_equal(dmu, (np.arange(6.0).reshape(3, 2) + [0.5, -2.0]).T)
    np.testing.assert_array_equal(ds2, [[-1.0, 0.0, -5.0], [-2.0, 0.0, -6.0]])
    with pytest.raises(ValueError, match="FSA"):
        gp.predict_f_grad(xs.T)
    with pytest.raises(ValueError):
        gp.predict_f_grad(xs.T, [[0, 3]])                       # an index outside the test points


def test_julia_fsa_dual_method_calls_the_entry_point():
    """the B200FSA Dual method passes nine arguments to gpb200_fitc_predict_fsa_grad, whose header declaration has nine"""
    src = open(os.path.join(ROOT, "gaussianprocesses.jl_b200", "julia", "GPB200.jl")).read()
    m = re.search(r"function predict_f\(gp::GPE\{[^}]*\}, x::DualMatrix, blockindpred::AbstractVector;[^\n]*CS<:B200FSA"
                  r".*?\nend\n", src, re.S)
    assert m, "no B200FSA Dual method"
    body = m.group(0)
    call = re.search(r"ccall\(\(:gpb200_fitc_predict_fsa_grad, LIB\), Cint,\s*\(([^)]*)\),\s*([^)]*)\)", body, re.S)
    assert call, "the method does not call gpb200_fitc_predict_fsa_grad"
    types = [t.strip() for t in call.group(1).split(",") if t.strip()]
    args = [a.strip() for a in call.group(2).split(",") if a.strip()]
    assert len(types) == 9 and len(args) == 9, (types, args)
    hdr = open(os.path.join(ROOT, "include", "gpb200.h")).read()
    decl = re.search(r"int\s+gpb200_fitc_predict_fsa_grad\(([^)]*)\);", hdr, re.S)
    assert decl and len(decl.group(1).split(",")) == 9
    assert "full_cov && throw(ArgumentError" in body and "dual_outputs(x, mu, dmu) .+ mean(gp.mean, x)" in body
