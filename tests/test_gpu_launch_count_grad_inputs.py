"""GPU: the launch counter of gpb200_grad_inputs against the kernels torch.profiler records (the
tests/test_gpu_launch_count_fitc_cv.py pattern): single GPU through both sweeps (SEIso specialisation and kernel program),
in the S state after gpa_grad, and a row-sharded in-process group, whose sum of the ranks' partials launches too.

The file sits with the other launch-count files: torch.profiler records no device activity in a session started about a
minute or more after the process's first profiling session (see test_gpu_tile_kernel_contracts.py), so the files that open
sessions must run next to each other."""
import numpy as np
import pytest

from conftest import make_data
from test_gpu_launch_count_fitc_cv import _device_kernels

pytestmark = pytest.mark.gpu


def test_grad_inputs_launch_count(tmp_path):
    import gpb200 as g
    X, y, _ = make_data(3000, 3, 81)
    rows = []
    for name, kern in (("SEIso", g.SEIso(0.2, 0.1)), ("SE+RQ", g.SEIso(0.2, 0.1) + g.RQIso(0.3, 0.0, 0.2))):
        gp = g.GPE(X.T, y, g.MeanZero(), kern, -1.0)
        e = gp._eng
        e.grad_prepare()
        v, dl = np.random.default_rng(82).standard_normal((2, 3000))
        steps = [("resident alpha", lambda: e.grad_inputs()), ("given alpha", lambda: e.grad_inputs(gp.alpha)),
                 ("S state", lambda: (e.gpa_grad(v, dl), e.grad_inputs()))]
        for step, fn in steps:
            c0 = e.launch_count()
            k = _device_kernels(fn, tmp_path)
            rows.append((name + " " + step, e.launch_count() - c0, k))
    grp = g.LocalGroupEngine(4, rb=1)
    try:
        gs = g.GPE(X.T, y, g.MeanZero(), g.SEIso(0.2, 0.1), -1.0, engine=grp)
        grp.grad_prepare()
        c0 = grp.launch_count()
        k = _device_kernels(lambda: grp.grad_inputs(), tmp_path)
        rows.append(("group of 4", grp.launch_count() - c0, k))
    finally:
        grp.close()
    for r in rows:
        print("launch count grad_inputs %-22s counted %6d  device %6d" % r)
    assert all(c == k for _, c, k in rows), rows
