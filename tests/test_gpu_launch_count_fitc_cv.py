"""GPU: the launch counter of the sparse engine's cross-validation entry points against the kernels torch.profiler records
(the tests/test_gpu_launch_count.py pattern): every kernel gpb200_fitc_get_inverse_diag / _cv_param / _cv_block enqueue is
counted in the wrapper that issues it.  Several row chunks (at most 32768 rows each), so a miscount inside the streaming loops
shows."""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _device_kernels(fn, tmp_path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "launches.pt.trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as fh:
        events = json.load(fh)["traceEvents"]
    return sum(1 for e in events if e.get("cat") == "kernel" and not e.get("name", "").startswith(("Memcpy", "Memset")))


@pytest.mark.parametrize("strategy", ["FITC", "SoR"])
def test_cv_launch_count(strategy, tmp_path):
    import gpb200 as g
    rng = np.random.default_rng(6)
    N, M, d = 70000, 60, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-2, 2, (M, d))
    gp = getattr(g, strategy)(X.T, Xu.T, y, g.MeanZero(), g.SEIso(-0.3, 0.0) + g.Noise(-1.0), -1.0)
    eng = gp._eng
    V = np.arange(0, N, 97)
    steps = [("inverse_diag", eng.inverse_diag), ("cv_param 0", lambda: eng.cv_param(0)), ("cv_block 1", lambda: eng.cv_block(1, V)),
             ("cv_param noise", lambda: eng.cv_param(-1)), ("cv_block 0", lambda: eng.cv_block(0, V)),
             ("cv_param Noise", lambda: eng.cv_param(2))]
    rows = []
    for name, fn in steps:
        c0 = eng.launch_count()
        kernels = _device_kernels(fn, tmp_path)
        rows.append((name, eng.launch_count() - c0, kernels))
    for r in rows:
        print("launch count %s %-16s counted %6d  device %6d" % (strategy, *r))
    assert all(c == k for _, c, k in rows), rows
