"""GPU: the launch counter of gpb200_fitc_grad_kernel_inducing and gpb200_fitc_set_inducing against the kernels
torch.profiler records (the tests/test_gpu_launch_count_fitc_cv.py pattern), for FITC, DTC, SoR and FSA.  The joint call issues grad_kernel's launches plus one contraction per chunk and one for W_uu.

The file sits with the other launch-count files: torch.profiler records no device activity in a session started about a
minute or more after the process's first profiling session, so the files that open sessions must run next to each other."""
import numpy as np
import pytest

from test_gpu_launch_count_fitc_cv import _device_kernels

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["FITC", "DTC", "SoR", "FSA"])
def test_inducing_launch_count(mode, tmp_path):
    import gpb200 as g
    rng = np.random.default_rng(21)
    N, M, d = 70000, 60, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-2, 2, (M, d))
    k = g.SEIso(-0.3, 0.0) + g.Noise(-1.0)
    if mode == "FSA":
        gp = g.FSA(X.T, Xu.T, [np.arange(i, min(i + 500, N)) for i in range(0, N, 500)], y, g.MeanZero(), k, -1.0)
    else:
        gp = getattr(g, mode)(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    e = gp._eng
    Xu2 = Xu + 0.01
    steps = [("grad_kernel", e.grad_kernel), ("grad_kernel_inducing", e.grad_kernel_inducing),
             ("grad_kernel_inducing no kernel", lambda: e.grad_kernel_inducing(want_kernel=False)),
             ("set_inducing", lambda: e.set_inducing(Xu2))]
    rows = []
    for name, fn in steps:
        c0 = e.launch_count()
        kern = _device_kernels(fn, tmp_path)
        rows.append((name, e.launch_count() - c0, kern))
    for r in rows:
        print("launch count %s %-32s counted %6d  device %6d" % (mode, *r))
    assert all(c == k for _, c, k in rows), rows
    assert rows[1][1] - rows[0][1] >= 2, rows                  # one contraction per staging chunk and one for W_uu
