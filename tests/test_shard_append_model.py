"""CPU: numpy model of append on ROW-SHARDED storage (shard_append / shard_append_solve in csrc/shard_impl.cuh), built on the
sharded-schedule model of test_shard_model.py.  Non-owned rows stay NaN, so a read outside the rows a rank owns (or outside the
blocks it received) poisons the result.  The rebuild starts at the ownership block b0 that holds the first touched tile:
  Gram rows >= b0 on their owners;  V = K[b0.., :b0] L11^-T solved like the test points of the sharded predict (the owner of
  each old column block solves and broadcasts it, keeps its transpose as the U part of its old rows, every rank applies it to
  its own later columns);  Schur complement of the own rows >= b0 with K = b0;  the sharded Cholesky from block b0 / NBp on."""
import numpy as np
import pytest

from test_shard_model import T, Model, _beyond_block_mask, nt


class AppendModel(Model):
    def cholesky(self, kb0=0):
        """Model.cholesky starting at block kb0 (the blocks before it are already factored)"""
        R = self.R
        for k in range(kb0, self.nblk):
            c0, nb, o = self.blk(k)
            r1 = c0 + nb
            Go = self.G[o]
            Lkk = np.linalg.cholesky(np.tril(Go[c0:r1, c0:r1]) + np.tril(Go[c0:r1, c0:r1], -1).T)
            self.F[o][c0:r1, c0:r1] = np.tril(Lkk) + np.triu(self.F[o][c0:r1, c0:r1], 1)
            stage_D = np.zeros((nb, T)); stage_DT = np.zeros((nb, T))
            for t in range(nb // T):
                W = np.linalg.inv(Lkk[t * T:(t + 1) * T, t * T:(t + 1) * T])
                stage_D[t * T:(t + 1) * T] = W
                stage_DT[t * T:(t + 1) * T] = W.T
            P = [np.full((self.Np, self.NB), np.nan) for _ in range(R)]
            for q in range(R):
                P[q][c0:r1, :nb] = np.tril(Lkk)
                self.Dinv[q][c0:r1] = stage_D; self.DinvT[q][c0:r1] = stage_DT
                self.logd[q][c0:r1] = 2.0 * np.log(np.diag(Lkk))
            S = [dict() for _ in range(R)]
            for q in range(R):
                rows = self.own_rows(q, r1)
                if rows:
                    self.trsm_rows(q, rows, c0, nb, P[q])
                    X = self.G[q][rows, c0:r1]
                    self.F[q][rows, c0:r1] = X
                    S[q].update(zip(rows, X))
            for q in range(R):
                for p in range(R):
                    for r, xr in S[p].items():
                        P[q][r, :nb] = xr
            self.F[o][c0:r1, r1:] = P[o][r1:, :nb].T
            for q in range(R):
                for i in self.own_rows(q, r1):
                    self.G[q][i, r1:i + 1] -= nt(P[q][i:i + 1, :nb], P[q][r1:i + 1, :nb])[0]

    def append(self, Kext, Nold, Nnew):
        R, NB = self.R, self.NB
        b0 = Nold // NB * NB
        Mv = -(-Nnew // T) * T - b0
        self.K = Kext
        # Gram rows >= b0 on their owners (lower part), identity beyond Nnew (Kext carries the padding)
        for q in range(R):
            for r in self.own_rows(q, b0):
                self.G[q][r, :r + 1] = Kext[r, :r + 1]
        if b0 == 0:
            return self.cholesky(0)
        # every rank: Kst = K[b0 .. b0+Mv, :b0]; columns beyond b0 are never read
        Kst = [np.full((Mv, self.Np), np.nan) for _ in range(R)]
        for q in range(R):
            Kst[q][:, :b0] = Kext[b0:b0 + Mv, :b0]
        for k in range(b0 // NB):
            c0, nb, o = self.blk(k)
            r1 = c0 + nb
            Pv = np.linalg.solve(np.tril(self.F[o][c0:r1, c0:r1]), Kst[o][:, c0:r1].T).T      # owner: block TRSM
            self.F[o][c0:r1, b0:b0 + Mv] = Pv.T                                               # U part of its old rows
            for q in range(R):                                                                 # broadcast, copy into Kst
                Kst[q][:, c0:r1] = Pv
                rows = self.own_rows(q, r1, b0)
                if rows:                                                                       # own later columns < b0
                    Kst[q][:, rows] -= nt(Pv, self.F[q][np.ix_(rows, range(c0, r1))])
        for q in range(R):
            rows = self.own_rows(q, b0, b0 + Mv)
            for r in rows:                                                                     # own rows of V -> rows of L
                self.F[q][r, :b0] = Kst[q][r - b0, :b0]
            for r in rows:                                                                     # Schur complement, K = b0
                self.G[q][r, b0:r + 1] -= nt(Kst[q][r - b0:r - b0 + 1, :b0], Kst[q][:r - b0 + 1, :b0])[0]
        assert all(np.array_equal(Kst[0][:, :b0], Kst[q][:, :b0]) for q in range(R))        # V is replicated
        self.cholesky(b0 // NB)


def _padded_gram(n, Np, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 3))
    K = np.eye(Np)
    K[:n, :n] = np.exp(-0.5 * ((X[:, None, :] - X[None, :, :]) ** 2).sum(-1)) + 0.3 * np.eye(n)
    return K


# (R, rb, n0, k): ownership block NB = 4 * rb rows; b0 = n0 // NB * NB
@pytest.mark.parametrize("R,rb,n0,k", [
    (2, 2, 3, 5),          # b0 = 0: first block, everything refactored
    (3, 2, 9, 1),          # b0 in block 1 (rank 1), k = 1
    (3, 2, 17, 6),         # block 2 (rank 2)
    (3, 2, 26, 4),         # block 3 (rank 0, second cycle)
    (3, 2, 13, 10),        # the new rows cross into the next block
    (2, 1, 16, 1),         # old N on a tile and block boundary
    (4, 1, 10, 9),         # rb = 1: every tile its own block
    (2, 4, 20, 30),        # wide blocks, k larger than a block
])
def test_sharded_append_model(R, rb, n0, k):
    n1 = n0 + k
    Np = -(-n1 // T) * T + T                        # capacity: one tile of padding beyond the new N
    Kext = _padded_gram(n1, Np, 11 * R + rb + n0)
    Kold = np.eye(Np)
    Kold[:n0, :n0] = Kext[:n0, :n0]
    m = AppendModel(Kold, R, rb)
    m.cholesky()
    m.append(Kext, n0, n1)
    L = np.linalg.cholesky(Kext)
    assert np.allclose(m.assembled(m.F, "lower"), L, atol=1e-12)
    assert np.allclose(np.triu(m.assembled(m.F, "upper"), 1), np.triu(L.T, 1) * _beyond_block_mask(m), atol=1e-12)
    assert all(np.array_equal(m.logd[0], lq) for lq in m.logd)
    assert abs(np.sum(m.logd[0]) - np.linalg.slogdet(Kext)[1]) < 1e-10
    rhs = np.random.default_rng(3).standard_normal(Np)
    assert np.allclose(m.solve(rhs), np.linalg.solve(Kext, rhs), atol=1e-10)
    m.inverse()
    assert np.allclose(m.assembled(m.G, "lower"), np.tril(np.linalg.inv(Kext)), atol=1e-10)


def test_append_model_reads_only_what_it_owns():
    """poisoning check of the model itself: a NaN planted in a row that no rank may read (an old row's stale Gram entry left
    of b0) does not reach the extended factor"""
    R, rb, n0, k = 3, 2, 17, 6
    Np = 28
    Kext = _padded_gram(n0 + k, Np, 5)
    Kold = np.eye(Np)
    Kold[:n0, :n0] = Kext[:n0, :n0]
    m = AppendModel(Kold, R, rb)
    m.cholesky()
    for q in range(R):
        for r in m.own_rows(q):
            m.G[q][r, :] = np.nan                   # the Schur complements of the first factorisation are dead
    m.append(Kext, n0, n0 + k)
    L = np.linalg.cholesky(Kext)
    assert np.allclose(m.assembled(m.F, "lower"), L, atol=1e-12)
