"""GPU: the launch counter of gpb200_fitc_grad_kernel_inputs and gpb200_fitc_set_inputs against the kernels torch.profiler
records (the tests/test_gpu_launch_count_fitc_cv.py pattern), for FITC, DTC, SoR and FSA.  The joint call issues the
launches of grad_kernel (or grad_kernel_inducing) plus one row contraction per staging chunk (FSA: plus one block
contraction per chunk); set_inputs launches nothing.

The file sits with the other launch-count files: torch.profiler records no device activity in a session started about a
minute or more after the process's first profiling session, so the files that open sessions must run next to each other."""
import numpy as np
import pytest

from test_gpu_launch_count_fitc_cv import _device_kernels

pytestmark = pytest.mark.gpu


def _chunks(N, M, blocks=None):
    """staging chunks of gpb200_fitc_set_data (modes 0-2) and of gpb200_fitc_set_blocks (FSA: whole padded blocks)"""
    Mpad = -(-M // 128) * 128
    cap = min(int(2.0e9 / (8.0 * Mpad)) // 128 * 128, 32768)
    if blocks is None:
        return -(-N // max(min(cap, -(-N // 128) * 128), 128))
    n, used = 1, 0
    for b in blocks:
        B = -(-len(b) // 128) * 128
        if used + B > cap:
            n, used = n + 1, 0
        used += B
    return n


@pytest.mark.parametrize("mode", ["FITC", "DTC", "SoR", "FSA"])
def test_inputs_launch_count(mode, tmp_path):
    import gpb200 as g
    rng = np.random.default_rng(22)
    N, M, d = 70000, 60, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1)) + 0.1 * rng.standard_normal(N)
    Xu = rng.uniform(-2, 2, (M, d))
    k = g.SEIso(-0.3, 0.0) + g.Noise(-1.0)
    blocks = [np.arange(i, min(i + 500, N)) for i in range(0, N, 500)] if mode == "FSA" else None
    if mode == "FSA":
        gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), k, -1.0)
    else:
        gp = getattr(g, mode)(X.T, Xu.T, y, g.MeanZero(), k, -1.0)
    e = gp._eng
    e.grad_kernel()                       # the sub-engines' inverses are now resident: every call below skips their build
    X2 = X + 0.01
    steps = [("grad_kernel", e.grad_kernel), ("grad_kernel_inputs", e.grad_kernel_inputs),
             ("grad_kernel_inputs no kernel", lambda: e.grad_kernel_inputs(want_kernel=False)),
             ("grad_kernel_inducing", e.grad_kernel_inducing),
             ("grad_kernel_inputs + Xu", lambda: e.grad_kernel_inputs(want_inducing=True)),
             ("set_inputs", lambda: e.set_inputs(X2))]
    rows = []
    for name, fn in steps:
        c0 = e.launch_count()
        kern = _device_kernels(fn, tmp_path)
        rows.append((name, e.launch_count() - c0, kern))
    for r in rows:
        print("launch count %s %-32s counted %6d  device %6d" % (mode, *r))
    assert all(c == k for _, c, k in rows), rows
    per_chunk = 2 if mode == "FSA" else 1
    added = per_chunk * _chunks(N, M, blocks)
    assert added >= 2
    assert rows[1][1] - rows[0][1] == added, rows
    assert rows[2][1] == rows[1][1]
    assert rows[4][1] - rows[3][1] == added, rows
    assert rows[5][1] == 0
