"""GPU: append for FITC, DTC and SoR (gpb200_fitc_append) against a fresh handle built on the concatenated data.  The appended
handle keeps Sigma_QR (rebuilt once as L_s L_s' after a factorize), adds the new rows' rank-k term and refactors; the fresh
handle streams every row.  Both reach the same M x M state by different sums, so the bounds are those of
tests/test_gpu_fitc_cv.py: max(1e-9, 64 cond(K_uu) cond(Sigma_QR) eps) of the largest entry."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LN = -1.0


def _kernel(kname):
    import gpb200 as g
    if kname == "SEIso":
        return g.SEIso(-0.5, 0.1)
    if kname == "Mat32+RQ":
        return g.Mat32Iso(-0.4, -0.1) + g.RQIso(0.2, -0.3, 0.1)
    return g.SEArd([-0.3, 0.1, -0.6], 0.05)


def _problem(n, m, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)
    Xu = rng.uniform(-2.0, 2.0, (m, d))
    return X, y, Xu


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _bound(spec, X, Xu, strategy):
    """(bound, cond(K_uu), cond(Sigma_QR)) with Sigma_QR formed densely in numpy"""
    m = Xu.shape[0]
    Kuu = orc.cov(spec, Xu) + 1e-10 * np.eye(m)
    Kuf = orc.cov(spec, Xu, X)
    s2 = math.exp(2.0 * LN)
    if strategy == "FITC":
        V = np.linalg.solve(np.linalg.cholesky(Kuu), Kuf)
        lam = s2 + orc._kdiag(spec, X) - np.sum(V * V, axis=0)
    else:
        lam = np.full(X.shape[0], s2)
    S = Kuu + (Kuf / lam) @ Kuf.T
    w, ws = np.linalg.eigvalsh(Kuu), np.linalg.eigvalsh(S)
    cu, cs = float(w[-1] / w[0]), float(ws[-1] / ws[0])
    return max(1e-9, 64.0 * cu * cs * EPS), cu, cs


def _model(strategy, kname, X, Xu, y):
    import gpb200 as g
    return getattr(g, strategy)(X.T, Xu.T, y, g.MeanZero(), _kernel(kname), LN)


def _compare(a, b, xs, full_r, checks_alpha=True):
    """every prediction right after the append, then (after mll with the full residuals) alpha, the gradients and CV"""
    ea, eb = a._eng, b._eng
    e = {"mll": _rel(a.mll, b.mll), "logdet": _rel(a.logdet, b.logdet)}
    ma, va = ea.predict(xs)
    mb, vb = eb.predict(xs)
    e["mu"], e["var"] = _rel(ma, mb), _rel(va, vb)
    e["cov"] = _rel(ea.predict_cov(xs[:64])[1], eb.predict_cov(xs[:64])[1])
    ga, gb = ea.predict_grad(xs), eb.predict_grad(xs)
    e["dmu"], e["dvar"] = _rel(ga[2], gb[2]), _rel(ga[3], gb[3])
    if checks_alpha:
        alpha, m, _ = ea.mll(full_r)
        e["mll(r)"] = _rel(m, b.mll)
        e["alpha"] = _rel(alpha, b.alpha)
        e["grad_noise"] = _rel(ea.grad_noise(), eb.grad_noise())
        e["grad_kernel"] = _rel(ea.grad_kernel(), eb.grad_kernel())
        e["inverse_diag"] = _rel(ea.inverse_diag(), eb.inverse_diag())
        za, zb = ea.cv_param(0), eb.cv_param(0)
        e["cv_param"] = max(_rel(za[0], zb[0]), _rel(za[1], zb[1]))
    return e


@pytest.mark.parametrize("k", [1, 127, 128, 129, 2500])
@pytest.mark.parametrize("kname", ["SEIso", "Mat32+RQ", "SEArd3"])
@pytest.mark.parametrize("strategy", ["FITC", "DTC", "SoR"])
def test_append_matches_a_fresh_handle(strategy, kname, k):
    n0, m, d = 1000, 100, 3                                   # staging chunk 1024 rows: k = 2500 takes three
    X, y, Xu = _problem(n0 + k, m, d, k + 7 * len(kname))
    xs = np.random.default_rng(5).standard_normal((300, d))
    a = _model(strategy, kname, X[:n0], Xu, y[:n0])
    a.append(X[n0:].T, y[n0:])
    assert a.alpha is None and a.nobs == n0 + k and a.target == a.mll
    b = _model(strategy, kname, X, Xu, y)
    tol, cu, cs = _bound(_kernel(kname).spec(), X, Xu, strategy)
    e = _compare(a, b, xs, y)
    print("%s %s k=%d cond(K_uu)=%.1e cond(Sigma_QR)=%.1e bound %.1e: %s"
          % (strategy, kname, k, cu, cs, tol, " ".join("%s %.1e" % kv for kv in e.items())))
    assert all(v <= tol for v in e.values()), e


@pytest.mark.parametrize("strategy", ["FITC", "SoR"])
def test_chained_appends_and_determinism(strategy):
    n0, m, d = 500, 80, 3
    rng = np.random.default_rng(3)
    sizes = rng.integers(1, 65, 200)
    X, y, Xu = _problem(n0 + int(sizes.sum()), m, d, 21)
    xs = rng.standard_normal((200, d))
    runs = []
    for _ in range(2):
        a = _model(strategy, "SEIso", X[:n0], Xu, y[:n0])
        r0 = n0
        for s in sizes:
            a.append(X[r0:r0 + s].T, y[r0:r0 + s])
            r0 += int(s)
        runs.append((a.mll, a.logdet) + a._eng.predict(xs) + (a,))
    (m1, l1, mu1, v1, a), (m2, l2, mu2, v2, _) = runs
    assert m1 == m2 and l1 == l2 and np.array_equal(mu1, mu2) and np.array_equal(v1, v2)      # bit for bit
    b = _model(strategy, "SEIso", X, Xu, y)
    tol, cu, cs = _bound(_kernel("SEIso").spec(), X, Xu, strategy)
    e = _compare(a, b, xs, y)
    print("chained %s N=%d cond(K_uu)=%.1e cond(Sigma_QR)=%.1e bound %.1e: %s"
          % (strategy, X.shape[0], cu, cs, tol, " ".join("%s %.1e" % kv for kv in e.items())))
    assert all(v <= tol for v in e.values()), e


def test_capacity_growth_releases_and_repeats_its_bytes():
    import gpb200 as g
    n0, m, d = 300, 64, 3
    X, y, Xu = _problem(n0 + 3000, m, d, 8)
    steps = [50, 700, 1, 1200, 49, 1000]                      # capacity 300 -> 600 -> 1200 -> 2400 -> 4800
    xs = np.random.default_rng(2).standard_normal((100, d))
    base = g.device_bytes()
    used = []
    for _ in range(2):
        a = _model("FITC", "SEIso", X[:n0], Xu, y[:n0])
        a._eng.grad_kernel(); a._eng.cv_param(0)              # workspaces sized at the first capacity
        r0 = n0
        for s in steps:
            a.append(X[r0:r0 + s].T, y[r0:r0 + s])
            r0 += s
        n = r0
        a._eng.mll(y[:n])
        used.append(g.device_bytes())
        b = _model("FITC", "SEIso", X[:n], Xu, y[:n])
        ea, eb = a._eng, b._eng
        tol, _, _ = _bound(_kernel("SEIso").spec(), X[:n], Xu, "FITC")
        ga, gb = ea.grad_kernel_inputs(want_inducing=True), eb.grad_kernel_inputs(want_inducing=True)
        e = {"dk": _rel(ga[0], gb[0]), "dxu": _rel(ga[1], gb[1]), "dx": _rel(ga[2], gb[2]),
             "inverse_diag": _rel(ea.inverse_diag(), eb.inverse_diag())}
        for j in (-1, 0, 1):
            za, zb = ea.cv_param(j), eb.cv_param(j)
            e["cv_param %d" % j] = max(_rel(za[0], zb[0]), _rel(za[1], zb[1]))
        V = np.arange(0, n, 37)
        e["cv_block"] = _rel(ea.cv_block(1, V), eb.cv_block(1, V))
        e["mu"] = _rel(ea.predict(xs)[0], eb.predict(xs)[0])
        print("growth N=%d bound %.1e: %s" % (n, tol, " ".join("%s %.1e" % kv for kv in e.items())))
        assert all(v <= tol for v in e.values()), e
        ea.close(); eb.close()
        assert g.device_bytes() == base
    assert used[0] == used[1]


def _raw_append(eng, k, x, ldx, r, mll=True):
    m, ld = C.c_double(), C.c_double()
    xp = x.ctypes.data_as(C.POINTER(C.c_double)) if x is not None else None
    rp = r.ctypes.data_as(C.POINTER(C.c_double)) if r is not None else None
    return eng._lib.gpb200_fitc_append(eng._h, k, xp, ldx, rp, C.byref(m) if mll else None, C.byref(ld)), m.value


def test_state_and_error_codes():
    import gpb200 as g
    from gpb200 import capi
    n0, m, d = 400, 50, 2
    X, y, Xu = _problem(n0 + 40, m, d, 4)
    xn, rn = np.ascontiguousarray(X[n0:n0 + 10]), y[n0:n0 + 10].copy()
    k = _kernel("SEIso")
    eng = capi.FitcEngine(0)
    eng.set_mode(0)
    eng.set_data(X[:n0], Xu)
    ops, dims, theta, _ = g.flatten(k, d)
    eng.set_kernel(ops, dims, theta.size)
    assert _raw_append(eng, 10, xn, d, rn)[0] == capi.ESTATE                      # before factorize
    eng.factorize(theta, LN)
    assert _raw_append(eng, 10, xn, d, rn)[0] == capi.ESTATE                      # before mll
    eng.mll(y[:n0])
    mu0, var0 = eng.predict(xn)
    for args in [(0, xn, d, rn), (-3, xn, d, rn), (10, xn, d - 1, rn), (10, None, d, rn), (10, xn, d, None)]:
        assert _raw_append(eng, *args)[0] == capi.EINVAL, args
    assert _raw_append(eng, 10, xn, d, rn, mll=False)[0] == capi.EINVAL
    bad = rn.copy(); bad[3] = np.nan
    assert _raw_append(eng, 10, xn, d, bad)[0] == capi.EINVAL
    bad[3] = np.inf
    assert _raw_append(eng, 10, xn, d, bad)[0] == capi.EINVAL
    mu1, var1 = eng.predict(xn)
    assert np.array_equal(mu0, mu1) and np.array_equal(var0, var1) and eng.N == n0         # nothing changed
    rc, mll = _raw_append(eng, 10, xn, d, rn)
    assert rc == capi.OK
    eng.N += 10
    mu2, _ = eng.predict(xn)                                                      # predictions right after the append
    for fn in (eng.grad_noise, eng.grad_kernel, eng.inverse_diag, lambda: eng.cv_param(0)):
        with pytest.raises(ValueError, match="mll first"):
            fn()
    _, m2, _ = eng.mll(y[:n0 + 10])
    assert abs(m2 - mll) <= 1e-9 * abs(mll)
    eng.grad_kernel(); eng.cv_param(0)
    eng.set_mode(3)                                                               # FSA: refused, handle usable afterwards
    assert _raw_append(eng, 10, np.ascontiguousarray(X[n0 + 10:n0 + 20]), d, y[n0 + 10:n0 + 20].copy())[0] == capi.EINVAL
    eng.set_mode(0)
    eng.factorize(theta, LN)
    eng.mll(y[:n0 + 10])
    mll3, _ = eng.append(X[n0 + 10:], y[n0 + 10:])
    ref = _model("FITC", "SEIso", X, Xu, y)
    assert abs(mll3 - ref.mll) <= 1e-9 * abs(ref.mll)
    assert _rel(eng.predict(xn)[0], ref._eng.predict(xn)[0]) <= 1e-9
    with pytest.raises(ValueError, match="FSA"):
        g.FSA(X[:n0].T, Xu.T, [np.arange(n0)], y[:n0], g.MeanZero(), _kernel("SEIso"), LN).append(xn.T, rn)


@pytest.mark.parametrize("what", ["set_inducing", "set_inputs", "factorize"])
def test_kept_sigma_qr_is_rebuilt_after(what):
    """an append, then a change that refactors, then another append: the second append must start from the new Sigma_QR"""
    n0, m, d = 600, 60, 3
    X, y, Xu = _problem(n0 + 200, m, d, 9)
    a = _model("FITC", "SEIso", X[:n0], Xu, y[:n0])
    a.append(X[n0:n0 + 100].T, y[n0:n0 + 100])
    rng = np.random.default_rng(1)
    if what == "set_inducing":
        Xu = Xu + 0.05 * rng.standard_normal(Xu.shape)
        a.set_params(np.concatenate([a.get_params(), Xu.ravel()]), inducing=True)
    elif what == "set_inputs":
        X = X.copy()
        X[:n0 + 100] += 0.05 * rng.standard_normal((n0 + 100, d))
        a.set_params(np.concatenate([a.get_params(), X[:n0 + 100].ravel()]), inputs=True)
    else:
        a.set_params(a.get_params() - 0.1)
    a.update_mll()
    a.append(X[n0 + 100:].T, y[n0 + 100:])
    b = _model("FITC", "SEIso", X, Xu, y)
    if what == "factorize":
        b.set_params(a.get_params()); b.update_mll()
    xs = rng.standard_normal((100, d))
    tol, _, _ = _bound(a.kernel.spec(), X, Xu, "FITC")
    e = _compare(a, b, xs, y)
    print("%s then append: bound %.1e: %s" % (what, tol, " ".join("%s %.1e" % kv for kv in e.items())))
    assert all(v <= tol for v in e.values()), e


@pytest.mark.slow
def test_large_append():
    """N = 10^6, M = 4096, SEIso d = 8: append 4096 rows against factorize + mll of the grown data.  cond(Sigma_QR) comes
    from Sigma_QR formed in torch on the device (the FITC Lambda by a triangular solve per row chunk)."""
    import torch
    import gpb200 as g
    n0, k, m, d = 1_000_000, 4096, 4096, 8
    rng = np.random.default_rng(0)
    X = rng.uniform(-2.0, 2.0, (n0 + k, d))                  # the workload of profiles/tools/fitc_append_bench.py
    y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n0 + k)
    Xu = X[rng.choice(n0, m, replace=False)]
    ll, lsig = math.log(0.8), 0.0
    kern = g.SEIso(ll, lsig)
    a = g.FITC(X[:n0].T, Xu.T, y[:n0], g.MeanZero(), kern, LN)
    a.append(X[n0:].T, y[n0:])
    b = g.FITC(X.T, Xu.T, y, g.MeanZero(), g.SEIso(ll, lsig), LN)
    dev = torch.device("cuda:0")
    U = torch.from_numpy(Xu).to(dev)
    sf2, l2 = math.exp(2 * lsig), math.exp(2 * ll)
    Kuu = sf2 * torch.exp(-0.5 * torch.cdist(U, U) ** 2 / l2) + 1e-10 * torch.eye(m, device=dev, dtype=torch.float64)
    Luu = torch.linalg.cholesky(Kuu)
    S = Kuu.clone()
    for r0 in range(0, n0 + k, 100_000):
        Xc = torch.from_numpy(X[r0:r0 + 100_000]).to(dev)
        Kuf = sf2 * torch.exp(-0.5 * torch.cdist(U, Xc) ** 2 / l2)
        V = torch.linalg.solve_triangular(Luu, Kuf, upper=False)
        lam = math.exp(2 * LN) + sf2 - (V * V).sum(0)
        S += (Kuf / lam) @ Kuf.T
    wu, ws = torch.linalg.eigvalsh(Kuu), torch.linalg.eigvalsh(S)
    cu, cs = float(wu[-1] / wu[0]), float(ws[-1] / ws[0])
    del S, Kuu, Luu, Kuf, V
    torch.cuda.empty_cache()
    tol = max(1e-9, 64.0 * cu * cs * EPS)
    xs = rng.uniform(-2.0, 2.0, (1024, d))
    (ma, va), (mb, vb) = a._eng.predict(xs), b._eng.predict(xs)
    e = {"mll": _rel(a.mll, b.mll), "logdet": _rel(a.logdet, b.logdet), "mu": _rel(ma, mb), "var": _rel(va, vb)}
    print("large append cond(K_uu)=%.1e cond(Sigma_QR)=%.1e bound %.1e: %s"
          % (cu, cs, tol, " ".join("%s %.1e" % kv for kv in e.items())))
    assert all(v <= tol for v in e.values()), e
