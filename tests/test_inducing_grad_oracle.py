"""CPU: the dense restatement of dmll/dXu (inducing_grad_oracle.dmll_dxu) against fourth-order central differences of the
oracle mll (gp_oracle.fitc_fit, fsa_oracle.fsa_fit) in every coordinate of Xu, for FITC, DTC, SoR and FSA over the
kernel zoo, and with Xu a subset of the training inputs for the smooth kernels."""
import numpy as np
import pytest

from conftest import kernel_zoo, make_data
import inducing_grad_oracle as ig

ZOO2 = [n for n, _ in kernel_zoo(2)]
# kernels that are smooth where an inducing point sits on a training input (no Mat12 kink, no Noise jump)
SMOOTH = ["SEIso", "SEArd", "Mat52Iso", "RQIso", "SE*RQ", "Poly", "LinIso+Const", "Periodic(1d)"]


# the linear-feature kernels have rank d + 1 (LinIso + Const) or (d + 1)(d + 2)/2 (degree-2 Poly): more inducing points than
# that leave K_uu singular up to its 1e-10 nugget and the mll without a meaningful derivative, so they get fewer
M_OF = {"LinIso+Const": 3, "Poly": 4}


def _spec(name, d):
    return dict(kernel_zoo(d))[name].spec()


def _blocks(n, seed):
    perm = np.random.default_rng(seed).permutation(n)
    cuts = [0, n // 3, n // 3 + 1, (3 * n) // 4, n]
    return [perm[cuts[i]:cuts[i + 1]] for i in range(len(cuts) - 1)]


def _check(spec, X, Xu, y, mode, blocks=None, ln=-1.0):
    """the closest of three steps: the mll's rounding grows with cond(Sigma_QR) (up to 1e7 here), the truncation error
    with the kernel's curvature (Periodic), so no single step serves the whole zoo"""
    g = ig.dmll_dxu(spec, X, Xu, y, ln, mode, blocks)
    scale = max(np.max(np.abs(g)), 1e-3)
    err = np.inf
    for h in (1e-3, 3e-4, 1e-4):
        err = min(err, np.max(np.abs(g - ig.fd_dmll_dxu(spec, X, Xu, y, ln, mode, blocks, h=h))))
        if err <= 1e-6 * scale:
            break
    assert err <= 1e-6 * scale, (mode, err, scale)
    return g


@pytest.mark.parametrize("mode", ig.MODES)
@pytest.mark.parametrize("name", ZOO2)
def test_dmll_dxu_fd_zoo(mode, name):
    d = 2
    X, y, _ = make_data(40, d, 11)
    Xu = np.random.default_rng(5).standard_normal((M_OF.get(name, 5), d)) * 1.2
    _check(_spec(name, d), X, Xu, y, mode, _blocks(40, 3) if mode == "FSA" else None)


@pytest.mark.parametrize("mode", ig.MODES)
@pytest.mark.parametrize("name", ["SEArd", "Masked", "MaunaLoa-like", "Fixed"])
def test_dmll_dxu_fd_d3(mode, name):
    d = 3
    X, y, _ = make_data(36, d, 12)
    Xu = np.random.default_rng(6).standard_normal((4, d))
    _check(_spec(name, d), X, Xu, y, mode, _blocks(36, 4) if mode == "FSA" else None)


@pytest.mark.parametrize("mode", ig.MODES)
@pytest.mark.parametrize("name", SMOOTH)
def test_dmll_dxu_fd_xu_subset_of_x(mode, name):
    """inducing points initialised at training inputs: the stationary leaves' derivative at r = 0 is the limit, 0"""
    d = 2
    X, y, _ = make_data(40, d, 13)
    Xu = X[::9][:M_OF.get(name, 5)].copy()
    _check(_spec(name, d), X, Xu, y, mode, _blocks(40, 5) if mode == "FSA" else None)


def test_fsa_one_point_blocks_equal_fitc():
    """singleton FSA blocks give FITC's Lambda up to the block nugget: the gradients agree to that order"""
    d = 2
    X, y, _ = make_data(30, d, 14)
    Xu = np.random.default_rng(7).standard_normal((4, d))
    spec = _spec("SEIso", d)
    g_fitc = ig.dmll_dxu(spec, X, Xu, y, -1.0, "FITC")
    g_fsa = ig.dmll_dxu(spec, X, Xu, y, -1.0, "FSA", [np.array([i]) for i in range(30)])
    assert np.max(np.abs(g_fitc - g_fsa)) <= 1e-7 * np.max(np.abs(g_fitc))
