"""GPU: the launch counter of gpb200_fitc_predict_fsa_grad against the kernels torch.profiler records (the
tests/test_gpu_launch_count_fitc_cv.py pattern): with and without the variance, in one test chunk and over several; and
the count does not depend on how many paired blocks share a training chunk.

The file sits with the other launch-count files: torch.profiler records no device activity in a session started about a
minute or more after the process's first profiling session (see test_gpu_tile_kernel_contracts.py), so the files that open
sessions must run next to each other."""
import numpy as np
import pytest

from test_gpu_launch_count_fitc_cv import _device_kernels

pytestmark = pytest.mark.gpu


def test_fsa_predict_grad_launch_count(tmp_path):
    import gpb200 as g
    rng = np.random.default_rng(41)
    N, M, d = 6000, 100, 2
    X = rng.standard_normal((N, d)); y = np.sin(X.sum(1))
    Xu = X[:M]
    order = np.argsort(X[:, 0])
    blocks = [order[i:i + 300] for i in range(0, N, 300)]
    gp = g.FSA(X.T, Xu.T, blocks, y, g.MeanZero(), g.SEIso(-0.5, 0.0) + g.RQIso(-0.3, -0.5, 0.2), -1.0)
    e = gp._eng
    Xs = np.ascontiguousarray(rng.standard_normal((400, d)))
    bo = np.where(np.arange(400) % 3 == 0, -1, np.arange(400) % len(blocks))
    Xbig = np.ascontiguousarray(rng.standard_normal((40000, d)))           # > one staging chunk of padded test rows
    bbig = np.full(40000, -1); bbig[:300] = np.arange(300) % len(blocks)
    one = np.zeros(4, dtype=np.int64)                                       # four points, one paired block ...
    four = np.arange(4, dtype=np.int64)                                     # ... or four blocks of the same training chunk
    steps = [("var", lambda: e.predict_fsa_grad(Xs, bo)), ("no var", lambda: e.predict_fsa_grad(Xs, bo, want_var=False)),
             ("var again", lambda: e.predict_fsa_grad(Xs, bo)), ("chunks", lambda: e.predict_fsa_grad(Xbig, bbig)),
             ("1 block", lambda: e.predict_fsa_grad(Xs[:4], one)), ("4 blocks", lambda: e.predict_fsa_grad(Xs[:4], four))]
    rows = []
    for name, fn in steps:
        c0 = e.launch_count()
        k = _device_kernels(fn, tmp_path)
        rows.append((name, e.launch_count() - c0, k))
    for r in rows:
        print("launch count predict_fsa_grad %-10s counted %6d  device %6d" % r)
    assert all(c == k for _, c, k in rows), rows
    assert rows[4][1] == rows[5][1]
    assert rows[3][1] > rows[0][1]                                          # several test chunks
