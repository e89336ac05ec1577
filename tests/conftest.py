import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussianprocesses.jl_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "slow: full-size property tests (minutes)")


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def engine():
    """One engine for the whole GPU session (fails loudly if the library or the GPU is missing)."""
    import gpb200
    eng = gpb200.Engine(0)
    yield eng
    eng.close()


def make_data(n, d, seed, m=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    y = np.sin(X.sum(axis=1)) + 0.1 * rng.standard_normal(n)
    Xs = rng.standard_normal((m, d)) if m else None
    return X, y, Xs


# kernel zoo: (name, constructor taking d) -- mirrors the list in test/kernels.jl:209-229
def kernel_zoo(d):
    import gpb200 as g
    ll = [0.1 * (i + 1) - 0.2 for i in range(d)]
    zoo = [
        ("SEIso", g.SEIso(0.3, 0.2)),
        ("SEArd", g.SEArd(ll, 0.1)),
        ("Mat12Iso", g.Mat12Iso(0.4, 0.1)),
        ("Mat32Iso", g.Mat32Iso(0.5, -0.1)),
        ("Mat52Iso", g.Mat52Iso(0.3, 0.2)),
        ("Mat12Ard", g.Mat12Ard(ll, 0.1)),
        ("Mat32Ard", g.Mat32Ard(ll, 0.2)),
        ("Mat52Ard", g.Mat52Ard(ll, -0.2)),
        ("RQIso", g.RQIso(0.4, 0.1, 0.3)),
        ("RQArd", g.RQArd(ll, 0.2, -0.3)),
        ("Periodic(1d)", g.Masked(g.Periodic(0.5, 0.1, 0.7), [0])),
        ("LinIso+Const", g.LinIso(0.6) + g.Const(-0.5)),
        ("LinArd+Noise", g.LinArd(ll) + g.Noise(-0.4)),
        ("Poly", g.Poly(0.2, -0.3, 2) + g.Const(0.1)),
        ("SE+RQ", g.SEIso(0.3, 0.1) + g.RQIso(0.5, -0.2, 0.1)),
        ("SE*RQ", g.SEIso(0.6, 0.1) * g.RQIso(0.5, 0.2, 0.1)),
        ("(SE+Mat12)*RQ", (g.SEIso(0.6, 0.1) + g.Mat12Iso(0.4, -0.2)) * g.RQIso(0.5, 0.2, 0.1)),
        ("Masked", g.Masked(g.SEIso(0.2, 0.1), [0]) + g.Masked(g.RQArd(ll[1:], 0.1, 0.2), list(range(1, d)))),
        ("Fixed", g.fix(g.RQIso(0.4, 0.1, 0.3), "lσ")),
        ("MaunaLoa-like", g.SEArd(ll, 0.0) + g.Masked(g.Periodic(0.0, 0.0, 0.3), [0]) * g.SEArd(ll, 0.0) + g.RQIso(0.0, 0.0, -1.0)
         + g.SEArd([v - 1.0 for v in ll], -1.0)),
    ]
    return zoo
