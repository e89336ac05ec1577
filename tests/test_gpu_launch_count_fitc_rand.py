"""GPU: the launch counter of gpb200_fitc_rand against the kernels torch.profiler records (the
tests/test_gpu_launch_count_fitc_cv.py pattern), for FITC, DTC, SoR and FSA: every kernel the call enqueues, the Ms x Ms
sub-engine's Cholesky included, is counted.  The first call creates the sub-engine, a second call at another Ms re-sizes it.

The file sits with the other launch-count files: torch.profiler records no device activity in a session started about a
minute or more after the process's first profiling session (see test_gpu_tile_kernel_contracts.py), so the files that open
sessions must run next to each other."""
import numpy as np
import pytest

from test_gpu_fitc_rand import MODES, _problem, _rand, _test_points
from test_gpu_launch_count_fitc_cv import _device_kernels

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", MODES)
def test_rand_launch_count(mode, tmp_path):
    gp, X, Xu, y, blocks = _problem(mode, "SEIso")
    Xs, bpred = _test_points(X, blocks, 300, seed=16)
    Xs2, bpred2 = _test_points(X, blocks, 700, seed=17)
    rng = np.random.default_rng(18)
    e = gp._eng
    rows = []
    for name, fn in [("rand 300", lambda: _rand(gp, Xs, bpred, 3, 1e-8, rng)), ("rand 700", lambda: _rand(gp, Xs2, bpred2, 3, 1e-8, rng)),
                     ("rand 700 again", lambda: _rand(gp, Xs2, bpred2, 3, 1e-8, rng))]:
        c0 = e.launch_count()
        k = _device_kernels(fn, tmp_path)
        rows.append((name, e.launch_count() - c0, k))
    for r in rows:
        print("launch count %s %-16s counted %6d  device %6d" % (mode, *r))
    assert all(c == k for _, c, k in rows), rows
