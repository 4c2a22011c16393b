"""TEST INFRASTRUCTURE ONLY -- dense oracle of the HD likelihood (``PulsarBatch.set_hd_likelihood``).

An independent restatement for small batches: it stacks every pulsar's noise covariance P_a (``os_oracle.dense_covariance``),
projected onto the null space G_a of its timing design matrix (SVD), into S0 = blockdiag(G_a^T P_a G_a), and the
common process into
    Fp = FG (A^2 Gamma (x) phi~) FG^T,   FG = blockdiag(G_a^T F_a),
whose cross-pulsar blocks are A^2 Gamma_ab G_a^T F_a phi~ F_b^T G_b.  Per grid point (A, gamma)
    ln L = 1/2 r^T S0^{-1} Fp S1^{-1} r - 1/2 ln det(I + S0^{-1} Fp),   S1 = S0 + Fp,  r -> stacked G_a^T r_a,
with dense solves and ``slogdet`` -- no Woodbury, no eigendecomposition.  Gamma of the named templates comes from
``os_oracle.hd_closed_form``.  Nothing here imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import curn_oracle as CO
from tests import os_oracle as OO


def orf_matrix(b, orf):
    """Gamma [P, P] of "hd", "monopole", "dipole" (diagonal 1) or a matrix, as given."""
    if not isinstance(orf, str):
        return np.asarray(orf, dtype=float)
    h, c = OO.hd_closed_form(b)
    return {"hd": h, "monopole": np.ones_like(h), "dipole": c}[orf]


def lnl_map(b, rows, log10_A, gamma, orf="hd", K=14, Tspan=None, models=None):
    """(ln L [R, Ng, NA], ln det(I + S0^{-1} Fp) [Ng, NA]) of engine-order rows [R, ld] by dense algebra."""
    if Tspan is None:
        Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    x, gam = np.atleast_1d(log10_A), np.atleast_1d(gamma)
    Gam = orf_matrix(b, orf)
    P, nc = b.n_psr, 2 * K
    blocks, bases, rs = [], [], []
    for i in range(P):
        n, s = b.ntoa[i], b.toa_off[i]
        G = CO.null_space(None if models is None else models[i], n)
        blocks.append(G.T @ OO.dense_covariance(b, i) @ G)
        bases.append(G.T @ OO.gw_basis(b.t_tdb[i], K, Tspan))
        rs.append(rows[:, s:s + n] @ G)
    m = [blk.shape[0] for blk in blocks]
    off = np.r_[0, np.cumsum(m)]
    S0 = np.zeros((off[-1], off[-1]))
    FG = np.zeros((off[-1], P * nc))
    for i in range(P):
        S0[off[i]:off[i + 1], off[i]:off[i + 1]] = blocks[i]
        FG[off[i]:off[i + 1], i * nc:(i + 1) * nc] = bases[i]
    r = np.concatenate(rs, axis=1)                                           # [R, n']
    a0 = np.linalg.solve(S0, r.T)
    out = np.zeros((rows.shape[0], len(gam), len(x)))
    ld = np.zeros((len(gam), len(x)))
    for g, gm in enumerate(gam):
        Sg = np.kron(Gam, np.diag(OO.phi_tilde(K, gm, Tspan)))              # [(a, i), (b, j)]
        for k, xa in enumerate(x):
            Fp = 10.0 ** (2 * xa) * (FG @ Sg @ FG.T)
            q = np.einsum("nr,nr->r", a0, Fp @ np.linalg.solve(S0 + Fp, r.T))
            sign, ld[g, k] = np.linalg.slogdet(np.eye(len(S0)) + np.linalg.solve(S0, Fp))
            assert sign > 0
            out[:, g, k] = 0.5 * q - 0.5 * ld[g, k]
    return out, ld


def lnl_of_statics(b, pc, ph, rows):
    """ln L [R, Ng, NA] from the plan's CURN projection C and HD statics (V, lambda, ldet) in numpy: the eigen form the
    kernel evaluates."""
    P, nc, ncp = b.n_psr, pc["nc"], pc["ncp"]
    X = np.zeros((rows.shape[0], P, ncp))
    for i in range(P):
        s, n = b.toa_off[i], b.ntoa[i]
        X[:, i, :nc] = rows[:, s:s + n] @ pc["C"][s:s + n, :nc]
    X = X.reshape(rows.shape[0], P * ncp)
    a2 = pc["a2"]
    y = np.einsum("gjk,rk->rgj", ph["V"], X)                                 # [R, Ng, np]
    w = a2[None, :, None] / (1.0 + a2[None, :, None] * ph["lam"][:, None, :])   # [Ng, NA, np]
    return 0.5 * np.einsum("rgj,gkj->rgk", y * y, w) - 0.5 * ph["ldet"][None]
