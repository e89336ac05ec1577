"""CPU: the dense restatement of dmll/dX for the sparse strategies (sparse_inputs_grad_oracle.dmll_dx) against fourth-order
central differences of the oracle mll (gp_oracle.fitc_fit, fsa_oracle.fsa_fit) in every coordinate of X, for FITC, DTC, SoR
and FSA: the kernel zoo at d = 1 and d = 3 (the Lin and Poly kernels exercise FITC's g_i term and the FSA blocks' diagonal),
MeanLin, training inputs on inducing points, and duplicated inputs inside an FSA block."""
import numpy as np
import pytest

from conftest import kernel_zoo, make_data
import sparse_inputs_grad_oracle as sg

ZOO1 = [n for n, _ in kernel_zoo(1)]
ZOO3 = [n for n, _ in kernel_zoo(3)]
# smooth where two points coincide: no Mat12 kink at r = 0, no Noise jump
SMOOTH = ["SEIso", "SEArd", "Mat52Iso", "RQIso", "SE*RQ", "Poly", "LinIso+Const", "Periodic(1d)"]
# the linear-feature kernels have low rank: more inducing points leave K_uu singular up to its nugget
M_OF = {"LinIso+Const": 2, "Poly": 3}


def _spec(name, d):
    return dict(kernel_zoo(d))[name].spec()


def _blocks(n, seed):
    perm = np.random.default_rng(seed).permutation(n)
    cuts = [0, 1, n // 3, (3 * n) // 4, n]
    return [perm[cuts[i]:cuts[i + 1]] for i in range(len(cuts) - 1)]


def _check(spec, X, Xu, y, mode, blocks=None, mspec=("MeanZero",), ln=-1.0):
    """the closest of three steps: the mll's rounding grows with cond(Sigma_QR), the truncation error with the kernel's
    curvature, so no single step serves the whole zoo"""
    g = sg.dmll_dx(spec, X, Xu, y, ln, mode, blocks, mspec)
    assert g.shape == X.shape and np.all(np.isfinite(g))
    scale = max(np.max(np.abs(g)), 1e-3)
    err = np.inf
    for h in (1e-3, 3e-4, 1e-4):
        err = min(err, np.max(np.abs(g - sg.fd_dmll_dx(spec, X, Xu, y, ln, mode, blocks, mspec, h=h))))
        if err <= 1e-6 * scale:
            break
    assert err <= 1e-6 * scale, (mode, err, scale)
    return g


@pytest.mark.parametrize("mode", sg.MODES)
@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("name", ZOO3)
def test_dmll_dx_fd_zoo(mode, d, name):
    if name not in ZOO1 and d == 1:
        pytest.skip("not in the d = 1 zoo")
    n = 9 if d == 1 else 6
    X, y, _ = make_data(n, d, 40 + d)
    Xu = np.random.default_rng(6 + d).standard_normal((M_OF.get(name, 3), d)) * 1.2
    _check(_spec(name, d), X, Xu, y, mode, _blocks(n, 3) if mode == "FSA" else None)


@pytest.mark.parametrize("mode", sg.MODES)
@pytest.mark.parametrize("name", ["SEIso", "Poly", "Masked"])
def test_dmll_dx_fd_linear_mean(mode, name):
    d = 3
    X, y, _ = make_data(7, d, 41)
    Xu = np.random.default_rng(8).standard_normal((M_OF.get(name, 3), d))
    spec, mspec = _spec(name, d), ("MeanLin", [0.4, -0.7, 0.2])
    blocks = _blocks(7, 4) if mode == "FSA" else None
    g = _check(spec, X, Xu, y, mode, blocks, mspec)
    assert np.max(np.abs(g - sg.dmll_dx(spec, X, Xu, y, -1.0, mode, blocks))) > 1e-3      # the mean's part is not empty


@pytest.mark.parametrize("mode", sg.MODES)
@pytest.mark.parametrize("name", SMOOTH)
def test_dmll_dx_fd_x_on_inducing_points(mode, name):
    """training inputs that coincide with inducing points: the stationary leaves' d1k at r = 0 is the limit, 0"""
    d = 2
    X, y, _ = make_data(9, d, 42)
    Xu = X[::3][:M_OF.get(name, 3)].copy()
    _check(_spec(name, d), X, Xu, y, mode, _blocks(9, 5) if mode == "FSA" else None)


@pytest.mark.parametrize("name", SMOOTH)
def test_dmll_dx_fd_fsa_duplicated_inputs_in_a_block(name):
    d = 2
    X, y, _ = make_data(9, d, 43)
    blocks = [np.array([0, 3, 7]), np.array([1, 2, 4, 5]), np.array([6, 8])]
    X[7] = X[3]                                                   # the same point twice in block 0
    Xu = np.random.default_rng(9).standard_normal((M_OF.get(name, 3), d))
    _check(_spec(name, d), X, Xu, y, "FSA", blocks)


def test_fitc_diagonal_term_is_the_total_derivative_of_k_ii():
    """LinIso: k(x, x) = |x|^2 / l^2 depends on x, so FITC's g_i term is not empty; without it the gradient is DTC's form"""
    d = 2
    X, y, _ = make_data(10, d, 44)
    Xu = np.random.default_rng(10).standard_normal((2, d))
    spec = ("LinIso", [0.1])
    g = _check(spec, X, Xu, y, "FITC")
    Guf, Gd, _ = sg.adjoints(spec, X, Xu, y, -1.0, "FITC")
    assert np.max(np.abs(np.diag(Gd))) > 1e-3
    import xgrad_oracle as xo
    g_rows = 0.5 * np.einsum("ji,ijp->ip", Guf, xo.cov_dx(spec, X, Xu)[1])
    assert np.max(np.abs(g - g_rows)) > 1e-3 * np.max(np.abs(g))


def test_fsa_one_point_blocks_equal_fitc():
    """singleton FSA blocks give FITC's Lambda up to the block nugget: the gradients agree to that order"""
    d = 2
    X, y, _ = make_data(12, d, 45)
    Xu = np.random.default_rng(11).standard_normal((3, d))
    spec = _spec("Poly", d)
    g_fitc = sg.dmll_dx(spec, X, Xu, y, -1.0, "FITC")
    g_fsa = sg.dmll_dx(spec, X, Xu, y, -1.0, "FSA", [np.array([i]) for i in range(12)])
    assert np.max(np.abs(g_fitc - g_fsa)) <= 1e-7 * np.max(np.abs(g_fitc))
