"""numpy model of the sparse engine's cross-validation schedule (gpb200_fitc_get_inverse_diag / _cv_param / _cv_block in
csrc/fitc_engine.cu): the same M x M state, the same two streaming passes over row chunks of `chunk` rows, the same row
epilogues.  Only K_uu^-1, S^-1 and per-chunk rows of K_fu / dK_fu are formed; the tests compare it against the dense
inverse of Sigma (tests/fitc_cv_oracle.py)."""
import math

import numpy as np

from oracle import gp_oracle as orc


class SparseCV:
    def __init__(self, spec, X, Xu, log_noise, mode="FITC", chunk=128):
        self.spec, self.X, self.Xu, self.mode, self.chunk = spec, np.asarray(X, float), np.asarray(Xu, float), mode, chunk
        m = self.Xu.shape[0]
        Kuu, self.gKuu = orc.cov_and_grads(spec, self.Xu, None, True)
        self.A = np.linalg.inv(Kuu + 1e-10 * np.eye(m))              # K_uu^-1 (the engine's first sub-engine)
        s2 = math.exp(2.0 * log_noise)
        n = self.X.shape[0]
        lam = np.empty(n)
        S = Kuu + 2e-10 * np.eye(m)                                    # Sigma_QR: K_uu + both nuggets
        for r0, K in self._chunks():
            q = np.einsum("ij,jk,ik->i", K, self.A, K)
            lam[r0:r0 + K.shape[0]] = s2 + orc._kdiag(spec, self.X[r0:r0 + K.shape[0]]) - q if mode == "FITC" else s2
            S += K.T @ (K / lam[r0:r0 + K.shape[0], None])
        self.lam, self.B = lam, np.linalg.inv(S)
        self.n_theta = len(self.gKuu)

    def _chunks(self, param=None):
        for r0 in range(0, self.X.shape[0], self.chunk):
            Xc = self.X[r0:r0 + self.chunk]
            if param is None:
                yield r0, orc.cov(self.spec, Xc, self.Xu)
            else:
                K, gK = orc.cov_and_grads(self.spec, Xc, self.Xu, True)
                yield r0, K, gK[param], Xc

    def inverse_diag(self):
        out = np.empty(self.X.shape[0])
        for r0, K in self._chunks():
            lam = self.lam[r0:r0 + K.shape[0]]
            out[r0:r0 + K.shape[0]] = 1.0 / lam - np.sum(K * (K @ self.B), axis=1) / lam ** 2
        return out

    def cv_param(self, param, alpha):
        """(Z_j alpha, diag(Z_j Sigma^-1)); param -1 = noise variance"""
        m, noise = self.Xu.shape[0], param < 0
        Dp = np.zeros((m, m)) if noise else self.gKuu[param] @ self.A
        R, H = np.zeros((m, m)), np.zeros((m, m))
        kta, gta, uD = np.zeros(m), np.zeros(m), np.zeros(m)
        delta = np.empty(self.X.shape[0])
        src = self._chunks(0 if noise else param)
        for r0, K, dK, Xc in src:                                     # pass 1
            sl = slice(r0, r0 + K.shape[0])
            lam, a = self.lam[sl], alpha[sl]
            G = np.zeros_like(K) if noise else dK - 0.5 * K @ Dp.T
            if noise:
                dl = np.ones(K.shape[0])
            elif self.mode == "FITC":
                dkd = np.array([orc.cov_and_grads(self.spec, Xc[i:i + 1], Xc[i:i + 1], True)[1][param][0, 0] for i in range(Xc.shape[0])])
                dl = dkd - 2.0 * np.sum(G * (K @ self.A), axis=1)
            else:
                dl = np.zeros(K.shape[0])
            delta[sl] = dl
            KL = K / lam[:, None]
            kta += K.T @ a
            uD += KL.T @ (dl * a)
            gta += G.T @ a
            R += KL.T @ G
            H += KL.T @ (KL * dl[:, None])
        beta = self.A @ kta
        w = gta - uD - R @ beta
        Q = H - R - R.T
        self._state = (param, Dp, Q, delta)
        zja, dg = np.empty(self.X.shape[0]), np.empty(self.X.shape[0])
        for r0, K, dK, Xc in self._chunks(0 if noise else param):     # pass 2
            sl = slice(r0, r0 + K.shape[0])
            lam, a, dl = self.lam[sl], alpha[sl], delta[sl]
            G = np.zeros_like(K) if noise else dK - 0.5 * K @ Dp.T
            Ch = (K @ self.B) / lam[:, None]
            P = Ch @ Q
            zja[sl] = dl * a / lam + (G @ beta) / lam + Ch @ w
            dg[sl] = dl / lam ** 2 + 2.0 * np.sum(G * Ch, axis=1) / lam - 2.0 * dl * np.sum(K * Ch, axis=1) / lam ** 2 + np.sum(P * Ch, axis=1)
        return zja, dg

    def cv_block(self, which, V):
        V = np.asarray(V)
        Xv, lam = self.X[V], self.lam[V]
        K, gK = orc.cov_and_grads(self.spec, Xv, self.Xu, True)
        Ch = (K @ self.B) / lam[:, None]
        if which == 0:
            return np.diag(1.0 / lam) - Ch @ (K / lam[:, None]).T
        param, Dp, Q, delta = self._state
        G = np.zeros_like(K) if param < 0 else gK[param] - 0.5 * K @ Dp.T
        E = 0.5 * Ch @ Q + G / lam[:, None] - (delta[V] / lam ** 2)[:, None] * K
        return np.diag(delta[V] / lam ** 2) + E @ Ch.T + Ch @ E.T
