"""TEST INFRASTRUCTURE ONLY -- dense oracle of the factorised free-spectrum likelihood (``PulsarBatch.set_free_spectrum``).

An independent restatement for small batches.  Per bin k and pulsar it builds the noise covariance P_a,k as an explicit
n_a x n_a matrix (``os_oracle.dense_covariance``, with the common process on the other bins' columns F_-k when one is
given), projects it onto the null space G of the timing design matrix (SVD) and forms Z_a[k] = F_k^T G S0^{-1} G^T F_k,
S0 = G^T P_a,k G.  Per grid point rho, for the stacked array (S0 = blockdiag, FG = blockdiag(G_a^T F_k,a)) and the ORF
Gamma (the identity for the uncorrelated model),
    ln L_k = 1/2 r^T S0^{-1} Fp S1^{-1} r - 1/2 ln det(I + S0^{-1} Fp),   Fp = rho^2 FG (Gamma (x) I_2) FG^T,  S1 = S0 + Fp,
with dense solves and ``slogdet`` -- no Woodbury on the basis, no eigendecomposition.  Nothing here imports the
product's statics code."""
from __future__ import annotations

import numpy as np

from tests import curn_oracle as CO
from tests import hd_oracle as HO
from tests import os_oracle as OO


def _tspan(b, Tspan):
    return max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb) if Tspan is None else Tspan


def blocks(b, k, K, Tspan=None, models=None, log10_A_common=None, gamma_common=13 / 3):
    """Per pulsar (S0 = G^T P_a,k G, FG = G^T F_k [n', 2], G) of bin k (0-based)."""
    Tspan = _tspan(b, Tspan)
    out = []
    for i in range(b.n_psr):
        n = b.ntoa[i]
        F = OO.gw_basis(b.t_tdb[i], K, Tspan)
        rest = np.r_[0:2 * k, 2 * k + 2:2 * K]
        P = OO.dense_covariance(b, i)
        if log10_A_common is not None and rest.size:
            phi = 10.0 ** (2 * log10_A_common) * OO.phi_tilde(K, gamma_common, Tspan)
            P = OO.dense_covariance(b, i, F[:, rest], phi[rest])
        G = CO.null_space(None if models is None else models[i], n)
        out.append((G.T @ P @ G, G.T @ F[:, 2 * k:2 * k + 2], G))
    return out


def z_blocks(b, K, **kw):
    """Z_a[k] [P, K, 2, 2] by dense solves."""
    Z = np.zeros((b.n_psr, K, 2, 2))
    for k in range(K):
        for i, (S0, FG, _) in enumerate(blocks(b, k, K, **kw)):
            Z[i, k] = FG.T @ np.linalg.solve(S0, FG)
    return 0.5 * (Z + Z.transpose(0, 1, 3, 2))


def lnl_map(b, rows, log10_rho, K, orf=None, **kw):
    """ln L [R, K, NR] of engine-order rows [R, ld]; ``orf`` None (uncorrelated) or a [P, P] matrix / template name."""
    x = np.atleast_1d(log10_rho)
    Gam = np.eye(b.n_psr) if orf is None else HO.orf_matrix(b, orf)
    out = np.zeros((rows.shape[0], K, len(x)))
    for k in range(K):
        bl = blocks(b, k, K, **kw)
        dims = [S0.shape[0] for S0, _, _ in bl]
        off = np.r_[0, np.cumsum(dims)]
        S0 = np.zeros((off[-1], off[-1]))
        FG = np.zeros((off[-1], 2 * b.n_psr))
        r = np.zeros((rows.shape[0], off[-1]))
        for i, (S, F, G) in enumerate(bl):
            S0[off[i]:off[i + 1], off[i]:off[i + 1]] = S
            FG[off[i]:off[i + 1], 2 * i:2 * i + 2] = F
            r[:, off[i]:off[i + 1]] = rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ G
        Fc = FG @ np.kron(Gam, np.eye(2)) @ FG.T
        a0 = np.linalg.solve(S0, r.T)
        for j, xr in enumerate(x):
            Fp = 10.0 ** (2 * xr) * Fc
            q = np.einsum("nr,nr->r", a0, Fp @ np.linalg.solve(S0 + Fp, r.T))
            sign, ld = np.linalg.slogdet(np.eye(len(S0)) + np.linalg.solve(S0, Fp))
            assert sign > 0
            out[:, k, j] = 0.5 * q - 0.5 * ld
    return out


def gather(b, pf, rows):
    """X_k [R, K, 2P] = the bin-k column pair of every pulsar's projection X_a = C_a^T r_a, from the plan's C."""
    K = len(pf["freqs"])
    X = np.zeros((rows.shape[0], K, 2 * b.n_psr))
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        Xa = rows[:, s:s + n] @ pf["C"][s:s + n, :2 * K]
        X[:, :, 2 * i:2 * i + 2] = Xa.reshape(-1, K, 2)
    return X


def lnl_of_statics(b, pf, rows, prefix=""):
    """ln L [R, K, NR] from the plan's statics (C, V, lambda, ldet) in numpy: the eigen form the kernel evaluates."""
    n = 2 * b.n_psr
    X = gather(b, pf, rows)
    V, lam, ldet = pf[prefix + "V"][:, :n, :n], pf[prefix + "lam"][:, :n], pf[prefix + "ldet"]
    a2 = pf["a2"]
    y = np.einsum("kji,rki->rkj", V, X)
    w = a2[None, :, None] / (1.0 + a2[None, :, None] * lam[:, None, :])          # [K, NR, n]
    return 0.5 * np.einsum("rkj,kij->rki", y * y, w) - 0.5 * ldet[None]
