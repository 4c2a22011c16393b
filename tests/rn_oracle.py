"""TEST INFRASTRUCTURE ONLY -- dense oracle of the single-pulsar red-noise likelihood
(``PulsarBatch.set_red_noise_likelihood``).

An independent restatement for small batches: per pulsar it builds the noise covariance P_a as an explicit n_a x n_a
matrix from the recipe the batch holds -- white variances, ECORR buckets and, when asked, a common power law on the
array-span basis; never the pulsar's own red noise, the model under test -- projects it onto the null space G of the
timing design matrix (SVD) and per grid point (A, gamma) evaluates, with F_a the (sin, cos) basis at k / T_a,
    ln L_a = 1/2 r^T S0^{-1} (G^T F_a phi_a F_a^T G) S1^{-1} r - 1/2 ln det(I + S0^{-1} G^T F_a phi_a F_a^T G),
    S0 = G^T P_a G,  S1 = S0 + G^T F_a phi_a F_a^T G,  r -> G^T r,
with dense solves and ``slogdet`` (the form of ``curn_oracle.lnl_map`` without the pulsar sum) -- no Woodbury, no
eigendecomposition.  ``summaries`` is ``curn_oracle.summaries`` on every (realization, pulsar) map.  Nothing here imports
the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import curn_oracle as CO
from tests import os_oracle as OO


def spans(b, Tspan=None):
    """T_a per pulsar: ``Tspan`` for every pulsar, or each pulsar's own t.max() - t.min()."""
    return [float(Tspan) if Tspan is not None else float(t.max() - t.min()) for t in b.t_tdb]


def covariance(b, i, log10_A_common=None, gamma_common=13 / 3, components_common=14):
    """P_a in engine order: white + ECORR (+ the common power law at k / Tspan of the array, k = 1..components_common)."""
    w1, w2 = b._white[i]
    P = np.diag(w1**2 + w2**2)
    if b._ecorr is not None and b._ecorr[i] is not None:
        bucket, e = b._ecorr[i]
        P = P + (np.asarray(e)[bucket] ** 2)[:, None] * (bucket[:, None] == bucket[None, :])
    if log10_A_common is not None:
        Tc = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
        Fc = OO.gw_basis(b.t_tdb[i], components_common, Tc)
        P = P + (Fc * 10.0 ** (2 * log10_A_common) * OO.phi_tilde(components_common, gamma_common, Tc)) @ Fc.T
    return P


def lnl_map(b, rows, log10_A, gamma, K=30, Tspan=None, models=None, **common):
    """ln L [R, P, Ng, NA] of engine-order rows [R, ld] by dense algebra; ``common``: the keyword arguments of
    ``covariance``."""
    x, gam = np.atleast_1d(log10_A), np.atleast_1d(gamma)
    out = np.zeros((rows.shape[0], b.n_psr, len(gam), len(x)))
    for i, Ta in enumerate(spans(b, Tspan)):
        n, s = b.ntoa[i], b.toa_off[i]
        G = CO.null_space(None if models is None else models[i], n)
        S0 = G.T @ covariance(b, i, **common) @ G
        FG = G.T @ OO.gw_basis(b.t_tdb[i], K, Ta)
        r = rows[:, s:s + n] @ G
        a0 = np.linalg.solve(S0, r.T)
        for g, gm in enumerate(gam):
            for k, xa in enumerate(x):
                Fp = (FG * 10.0 ** (2 * xa) * OO.phi_tilde(K, gm, Ta)) @ FG.T
                q = np.einsum("nr,nr->r", a0, Fp @ np.linalg.solve(S0 + Fp, r.T))
                sign, ld = np.linalg.slogdet(np.eye(len(S0)) + np.linalg.solve(S0, Fp))
                assert sign > 0
                out[:, i, g, k] = 0.5 * q - 0.5 * ld
    return out


def ldet(b, log10_A, gamma, K=30, Tspan=None, models=None, **common):
    """[P, Ng, NA] ln det(I + S0^{-1} G^T F_a phi_a F_a^T G) by ``slogdet``."""
    x, gam = np.atleast_1d(log10_A), np.atleast_1d(gamma)
    out = np.zeros((b.n_psr, len(gam), len(x)))
    for i, Ta in enumerate(spans(b, Tspan)):
        G = CO.null_space(None if models is None else models[i], b.ntoa[i])
        S0 = G.T @ covariance(b, i, **common) @ G
        FG = G.T @ OO.gw_basis(b.t_tdb[i], K, Ta)
        for g, gm in enumerate(gam):
            for k, xa in enumerate(x):
                Fp = (FG * 10.0 ** (2 * xa) * OO.phi_tilde(K, gm, Ta)) @ FG.T
                out[i, g, k] = np.linalg.slogdet(np.eye(len(S0)) + np.linalg.solve(S0, Fp))[1]
    return out


def summaries(lnl, log10_A, gamma, kind="log-uniform", ul=0.95):
    """``curn_oracle.summaries`` of every map of lnl [R, P, Ng, NA]; every output gains the leading [R, P] axes."""
    R, P, NG, NA = lnl.shape
    s = CO.summaries(lnl.reshape(R * P, NG, NA), log10_A, gamma, kind, ul)
    return {k: v.reshape((R, P) + v.shape[1:]) for k, v in s.items()}


def lnl_of_statics(b, pr, rows):
    """ln L [R, P, Ng, NA] from the plan's statics (C, V, lambda, ldet) in numpy: the eigen form the kernels evaluate."""
    nc, a2 = pr["nc"], pr["a2"]
    out = np.zeros((rows.shape[0], b.n_psr, len(pr["gamma"]), len(a2)))
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        X = rows[:, s:s + n] @ pr["C"][s:s + n, :nc]                        # [R, nc]
        y = np.einsum("gji,ri->rgj", pr["V"][i][:, :nc, :nc], X)           # [R, Ng, nc]
        w = a2[None, :, None] / (1.0 + a2[None, :, None] * pr["eig"][i][:, None, :])   # [Ng, NA, nc]
        out[:, i] = 0.5 * np.einsum("rgj,gkj->rgk", y * y, w) - 0.5 * pr["ldet"][i][None]
    return out
