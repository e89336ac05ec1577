"""CPU: the descriptor model of the NT GEMM (tests/gemm_model.py).

1. The port of decode_tile's rasterisation enumerates exactly the model's tile set (plain grouped walk, lower trapezoid,
   compact owned-row grid and the filtered grid of batched ownership launches).
2. Driven by the descriptors the engine issues (transcribed from csrc/gpb200.cu), the model reproduces inv(L), tril(K^-1),
   the leaf panel TRSM and the Schur complement of a numpy factor, with every buffer element the model says is not read
   poisoned with NaN.  This ties the model, and so the GPU contract tests built on it, to what the engine assumes."""
import itertools

import numpy as np
import pytest

import gemm_model as gm
from gemm_model import KHI_M, KHI_N, KLO_M, KLO_N, LOWER_ONLY, SKIP_FIRST, Desc, Operand

T = gm.BM


def _check_bijection(d):
    got, have = gm.rasterised_tiles(d)
    assert len(got) == len(set(got)), "a tile is computed twice"
    assert set(got) == have


@pytest.mark.parametrize("GM_flag", [0, KLO_M])            # GROUP_M 16 and GM_TRI = 4
@pytest.mark.parametrize("lower", [False, True])
def test_rasterisation_is_a_bijection_onto_the_tile_set(GM_flag, lower):
    sizes = (1, 2, 3, 4, 5, 15, 16, 17, 20, 21, 33, 47, 64, 69, 70)
    for tm, tn in itertools.product(sizes, sizes):
        if lower and tn > tm:
            continue
        _check_bijection(Desc(Operand("A"), Operand("B"), "C", M=tm * T, N=tn * T, K=T,
                              flags=GM_flag | (LOWER_ONLY if lower else 0)))


@pytest.mark.parametrize("lower", [False, True])
def test_owned_row_grids_are_a_bijection_onto_the_tile_set(lower):
    for tm, tn, mod, div in itertools.product((1, 7, 20, 33), (1, 3, 7), (2, 3, 8), (1, 2, 4)):
        if lower and tn > tm:
            continue
        for off, rem in itertools.product((0, 1, 5, 12), range(mod)):
            flags = LOWER_ONLY | KLO_M if lower else 0
            kw = dict(M=tm * T, N=tn * T, K=T, flags=flags, bm_mod=mod, bm_rem=rem, bm_div=div, bm_off=off)
            _check_bijection(Desc(Operand("A"), Operand("B"), "C", **kw))                  # compact grid (batch 1)
            _check_bijection(Desc(Operand("A"), Operand("B"), "C", batch=2, zstep=T, **kw))  # filtered grid


def test_model_k_ranges_follow_the_flags():
    d = Desc(Operand("A"), Operand("B"), "C", M=3 * T, N=3 * T, K=3 * T, flags=KLO_M | KHI_N, klo_off=32)
    rng = {(t.bm, t.bn): (t.klo, t.khi) for t in gm.tiles(d)}
    assert rng[(0, 0)] == (32, 128) and rng[(1, 2)] == (160, 384) and rng[(2, 0)] == (288, 128)
    d = Desc(Operand("A"), Operand("B"), "C", M=2 * T, N=2 * T, K=4 * T, flags=KLO_N | KHI_M, k_lim=3 * T)
    assert {(t.bm, t.bn): (t.klo, t.khi) for t in gm.tiles(d)} == {(0, 0): (0, 128), (0, 1): (128, 128),
                                                                    (1, 0): (0, 256), (1, 1): (128, 256)}


# ---- engine schedules ------------------------------------------------------------------------------------------------

def _spd(Np, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((Np, Np))
    return X @ X.T / Np + np.eye(Np)


def _leaf_outputs(L, Np):
    Dinv = np.zeros((Np, T))
    for p in range(0, Np, T):
        Dinv[p:p + T] = np.linalg.inv(L[p:p + T, p:p + T])
    Dinv = np.tril(Dinv.reshape(-1, T, T)).reshape(Np, T)
    DinvT = np.concatenate([b.T for b in Dinv.reshape(-1, T, T)])
    return Dinv, DinvT


def _merge_inverse(Np, p, n1, n2, batch):
    """merge_inverse (gpb200.cu)"""
    lim = Np - p - n1
    return [Desc(Operand("G", "DinvT", p, p), Operand("F", None, p + n1, p), "F", c_row0=p, c_col0=p + n1,
                 M=n1, N=n2, K=n1, flags=KLO_M, batch=batch, zstep=2 * n1, n_lim=lim),
            Desc(Operand("G", "Dinv", p + n1, p + n1), Operand("F", None, p, p + n1), "G", c_row0=p + n1, c_col0=p,
                 Ct="G", ct_row0=p, ct_col0=p + n1, M=n2, N=n1, K=n2, alpha=-1.0, flags=KHI_M, batch=batch,
                 zstep=2 * n1, m_lim=lim, k_lim=lim)]


def _inverse_from_factor(Np):
    """inverse_merges + inverse_from_factor (gpb200.cu)"""
    out = []
    s = T
    while s < Np:
        out += _merge_inverse(Np, 0, s, min(Np - s, s), (Np + 2 * s - 1) // (2 * s))
        s *= 2
    return out, Desc(Operand("G", "DinvT"), Operand("G", "DinvT"), "G", M=Np, N=Np, K=Np, flags=LOWER_ONLY | KLO_M)


def _run_poisoned(descs, bufs):
    """Run the schedule once to learn which initial elements it reads, then again from buffers where every other element
    is NaN.  Returns the buffers of the second run."""
    probe = {k: v.copy() for k, v in bufs.items()}
    seen = {k: np.zeros(v.shape, bool) for k, v in bufs.items()}
    written = {k: np.zeros(v.shape, bool) for k, v in bufs.items()}
    for d in descs:
        r, w = gm.run(d, probe)
        for k in bufs:
            seen[k] |= r[k] & ~written[k]
            written[k] |= w[k]
    out = {k: np.where(seen[k], v, np.nan) for k, v in bufs.items()}
    for d in descs:
        gm.run(d, out)
    return out, written


@pytest.mark.parametrize("Np", [640, 1024])
def test_engine_inverse_schedule_reproduces_inv_L_and_tril_Kinv(Np):
    K = _spd(Np, Np)
    L = np.linalg.cholesky(K)
    Dinv, DinvT = _leaf_outputs(L, Np)
    merges, wtw = _inverse_from_factor(Np)
    bufs = dict(F=np.tril(L), G=np.full((Np, Np), np.nan), Dinv=Dinv, DinvT=DinvT)
    after, _ = _run_poisoned(merges, bufs)
    W = np.tril(after["G"], -1)
    for p in range(0, Np, T):
        W[p:p + T, p:p + T] = Dinv[p:p + T]
    Wref = np.linalg.inv(L)
    assert np.max(np.abs(W - Wref)) <= 1e-12 * np.max(np.abs(Wref))
    assert np.array_equal(np.triu(after["G"], T), np.tril(after["G"], -T).T)     # Ct: W' in the strict-upper tiles
    after, written = _run_poisoned(merges + [wtw], bufs)
    Kinv = np.linalg.inv(K)
    low = np.tril(np.ones((Np, Np), bool))
    assert np.max(np.abs(after["G"][low] - Kinv[low])) <= 1e-12 * np.max(np.abs(Kinv))
    # the upper halves of the diagonal tiles are never written
    for p in range(0, Np, T):
        assert not written["G"][p:p + T, p:p + T][np.triu_indices(T, 1)].any()


def test_engine_panel_trsm_and_schur_update_reproduce_the_factor():
    Np, p, k = 640, 0, 256
    K = _spd(Np, 7)
    L = np.linalg.cholesky(K)
    Dinv, _ = _leaf_outputs(L, Np)
    # panel_trsm_leaf (gpb200.cu): F[r0.., p..p+128) = G[r0.., p..p+128) W_pp'
    d = Desc(Operand("G", None, T, p), Operand("Dinv", None, p, 0), "F", c_row0=T, c_col0=p, M=Np - T, N=T, K=T)
    after, _ = _run_poisoned([d], dict(G=np.tril(K), F=np.full((Np, Np), np.nan), Dinv=Dinv))
    assert np.max(np.abs(after["F"][T:, :T] - L[T:, :T])) <= 1e-12 * np.max(np.abs(L))

    def schur(r0, rows, cols, extra=0):          # schur_update (gpb200.cu)
        return Desc(Operand("F", None, r0, p), Operand("F", None, r0, p), "G", c_row0=r0, c_col0=r0,
                    M=rows, N=cols, K=k, alpha=-1.0, beta=1.0, flags=LOWER_ONLY | extra)

    r0, rows = p + k, Np - p - k
    S = K[r0:, r0:] - L[r0:, :k] @ L[r0:, :k].T
    for sched in ([schur(r0, rows, rows)],
                  [schur(r0, T, T), schur(r0, rows, rows, SKIP_FIRST)],          # look-ahead split (chol_panel)
                  [schur(r0, rows, 2 * T), schur(r0 + 2 * T, rows - 2 * T, rows - 2 * T)]):   # trapezoid, then the rest
        after, written = _run_poisoned(sched, dict(F=np.tril(L), G=np.where(np.tri(Np, dtype=bool), K, np.nan)))
        got = after["G"][r0:, r0:]
        low = np.tri(rows, dtype=bool)
        assert np.max(np.abs(got[low] - S[low])) <= 1e-12 * np.max(np.abs(S))
        assert np.isnan(got[~low]).all()


def test_model_rejects_overlapping_reads_and_writes():
    bufs = dict(G=np.zeros((256, 256)))
    with pytest.raises(AssertionError):
        gm.run(Desc(Operand("G"), Operand("G"), "G", M=256, N=256, K=256), bufs)
