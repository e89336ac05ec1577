"""GPU: the launch counter of gpb200_predict_grad against the kernels torch.profiler records (the
tests/test_gpu_launch_count_fitc_cv.py pattern): with and without the variance, in one chunk and in three.

The file sits with the other launch-count files: torch.profiler records no device activity in a session started about a
minute or more after the process's first profiling session (see test_gpu_tile_kernel_contracts.py), so the files that open
sessions must run next to each other."""
import numpy as np
import pytest

from conftest import make_data
from test_gpu_launch_count_fitc_cv import _device_kernels

pytestmark = pytest.mark.gpu


def test_predict_grad_launch_count(tmp_path, monkeypatch):
    import gpb200 as g
    X, y, _ = make_data(3000, 3, 71)
    gp = g.GPE(X.T, y, g.MeanZero(), g.SEIso(0.2, 0.1) + g.RQIso(0.3, 0.0, 0.2), -1.0)
    Xs = np.random.default_rng(72).standard_normal((300, 3))
    e = gp._eng
    steps = [("var", lambda: e.predict_grad(Xs)), ("no var", lambda: e.predict_grad(Xs, want_var=False)),
             ("var again", lambda: e.predict_grad(Xs))]
    rows = []
    for name, fn in steps:
        c0 = e.launch_count()
        k = _device_kernels(fn, tmp_path)
        rows.append((name, e.launch_count() - c0, k))
    monkeypatch.setenv("GPB200_PREDICT_CHUNK", "128")
    c0 = e.launch_count()
    k = _device_kernels(lambda: e.predict_grad(Xs), tmp_path)
    rows.append(("3 chunks", e.launch_count() - c0, k))
    for r in rows:
        print("launch count predict_grad %-10s counted %6d  device %6d" % r)
    assert all(c == k for _, c, k in rows), rows
