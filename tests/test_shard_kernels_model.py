"""CPU: the index model tests/shard_kernels_model.py that test_gpu_shard_kernel_contracts.py holds the kernels to, checked
against brute-force enumeration, so that a slip in the model cannot hide one in a kernel."""
import numpy as np
import pytest

import shard_kernels_model as sm

T = sm.T


@pytest.mark.parametrize("R,rb", sm.LAYOUTS)
def test_own_before_and_compact_rows_enumerate_the_owned_tiles(R, rb):
    for n_tiles in sm.tile_counts(R, rb):
        seen = []
        for me in range(R):
            for t in range(n_tiles + 1):
                assert sm.own_before(t, me, R, rb) == sum(1 for u in range(t) if sm.owner(u, R, rb) == me)
            rows = sm.compact_rows(n_tiles, me, R, rb)
            assert np.array_equal(rows, np.flatnonzero(sm.own_row_mask(n_tiles * T, me, R, rb)))
            assert rows.size == sm.own_rows(n_tiles * T, me, R, rb) == sm.own_rows(n_tiles * T - 37, me, R, rb)
            # compact index of own row r of tile t: own_before(t) * 128 + r % 128 (shard_kernels.cuh)
            li = np.array([sm.own_before(r // T, me, R, rb) * T + r % T for r in rows], np.int64)
            assert np.array_equal(li, np.arange(rows.size))
            for t1 in range(n_tiles + 1):
                sub = sm.compact_rows(n_tiles, me, R, rb, t1)
                assert np.array_equal(sub, rows[rows >= t1 * T])
            seen.append(rows)
        allrows = np.sort(np.concatenate(seen))
        assert np.array_equal(allrows, np.arange(n_tiles * T))          # every row has exactly one owner


@pytest.mark.parametrize("R", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("tiles", [2, 3, 5, 8, 9, 12, 17])
def test_slices_partition_every_w21_block(R, tiles):
    Np = tiles * T
    for s in sm.split_levels(Np, R):
        assert s % (T * R) == 0 and s < Np
        cols = np.sort(np.concatenate([sm.slice_cols(s, R, q) for q in range(R)]))
        assert np.array_equal(cols, np.arange(s))
        rows = 0
        for z, p, n2 in sm.problems(s, Np):
            assert p == 2 * s * z and 0 < n2 <= s and p + s + n2 <= Np
            rows += n2
        assert sm.per_rank(s, Np, R) == rows * (s // R)
    # inverse_dist's rule: a level is split when its tile count is a positive multiple of R
    want = [s for s in (T << k for k in range(12)) if s < Np and (s // T) % R == 0]
    assert sm.split_levels(Np, R) == want
