"""TEST INFRASTRUCTURE ONLY -- dense oracle of the CURN likelihood (``PulsarBatch.set_curn_likelihood``).

An independent restatement for small batches: per pulsar it builds the noise covariance P_a as an explicit n_a x n_a
matrix (``os_oracle.dense_covariance``), projects it onto the null space G of the timing design matrix (SVD), and per
grid point (A, gamma) evaluates
    ln L = 1/2 r^T S0^{-1} (G^T F phi F^T G) S1^{-1} r - 1/2 ln det(I + S0^{-1} G^T F phi F^T G)
         (= 1/2 r^T S0^{-1} r - 1/2 r^T S1^{-1} r, without the cancellation),
    S0 = G^T P_a G,  S1 = S0 + G^T F phi F^T G,  r -> G^T r,
with dense solves and ``slogdet`` -- no Woodbury, no eigendecomposition.  ``summaries`` reduces a map to the grid
summaries with its own trapezoid weights and prior.  Nothing here imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def null_space(M, n):
    """G [n, n - rank]: orthonormal null space of M^T (identity without a model)."""
    if M is None:
        return np.eye(n)
    U, s, _ = np.linalg.svd(M, full_matrices=True)
    return U[:, int(np.sum(s > 1e-10 * s[0])):]


def lnl_map(b, rows, log10_A, gamma, K=14, Tspan=None, models=None):
    """ln L [R, Ng, NA] of engine-order rows [R, ld] by dense algebra."""
    if Tspan is None:
        Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    x, gam = np.atleast_1d(log10_A), np.atleast_1d(gamma)
    out = np.zeros((rows.shape[0], len(gam), len(x)))
    for i in range(b.n_psr):
        n, s = b.ntoa[i], b.toa_off[i]
        G = null_space(None if models is None else models[i], n)
        S0 = G.T @ OO.dense_covariance(b, i) @ G
        FG = G.T @ OO.gw_basis(b.t_tdb[i], K, Tspan)
        r = rows[:, s:s + n] @ G                                             # [R, n']
        a0 = np.linalg.solve(S0, r.T)
        for g, gm in enumerate(gam):
            for k, xa in enumerate(x):
                phi = 10.0 ** (2 * xa) * OO.phi_tilde(K, gm, Tspan)
                Fp = (FG * phi) @ FG.T
                # r^T (S0^-1 - S1^-1) r = r^T S0^-1 Fp S1^-1 r: the same quantity without the cancellation
                q = np.einsum("nr,nr->r", a0, Fp @ np.linalg.solve(S0 + Fp, r.T))
                sign, ld = np.linalg.slogdet(np.eye(len(S0)) + np.linalg.solve(S0, Fp))
                assert sign > 0
                out[:, g, k] += 0.5 * q - 0.5 * ld
    return out


def weights(v):
    """Trapezoid weights, restated: (v_{k+1} - v_{k-1}) / 2 inside, half an interval at the ends, 1 for one node."""
    v = np.asarray(v, dtype=float)
    if v.size == 1:
        return np.ones(1)
    w = np.empty(v.size)
    w[0], w[-1] = (v[1] - v[0]) / 2, (v[-1] - v[-2]) / 2
    w[1:-1] = (v[2:] - v[:-2]) / 2
    return w


def prior(log10_A, gamma, kind):
    """Prior density on the grid [NA], normalised so that sum_g sum_k w_g w_k pi_k = 1."""
    p = np.ones(len(log10_A)) if kind == "log-uniform" else 10.0 ** np.asarray(log10_A, dtype=float)
    return p / (weights(gamma).sum() * np.sum(weights(log10_A) * p))


def summaries(lnl, log10_A, gamma, kind="log-uniform", ul=0.95):
    """Grid summaries of maps [R, Ng, NA]: lnL_max, ml_gamma_index, ml_log10_A_index (first argmax, gamma-major),
    ln_bayes, post_log10_A [R, NA], post_gamma [R, Ng], log10_A_ul (the ``ul`` quantile of the trapezoid CDF of
    post_log10_A, normalised by its last node, linear between nodes)."""
    R, NG, NA = lnl.shape
    x = np.asarray(log10_A, dtype=float)
    wg, wx, pi = weights(gamma), weights(x), prior(x, gamma, kind)
    flat = lnl.reshape(R, -1)
    am = np.argmax(flat, axis=1)
    m = flat[np.arange(R), am]
    e = np.exp(lnl - m[:, None, None])
    # B in two stages (gamma, then log10 A): one flat einsum over the NG x NA map accumulates a rounding error of
    # ~ NG NA u (1e-12 at 256 x 256), more than the summaries it is the yardstick for
    S = np.einsum("g,rgk->rk", wg, e)
    B = S @ (wx * pi)
    post_a = S * pi / B[:, None]
    post_g = np.einsum("k,rgk->rg", wx * pi, e) / B[:, None]
    ulv = np.empty(R)
    for r in range(R):
        cdf = np.r_[0.0, np.cumsum(0.5 * np.diff(x) * (post_a[r, 1:] + post_a[r, :-1]))]
        t = ul * cdf[-1]
        k = int(np.argmax(cdf >= t))
        ulv[r] = x[k - 1] + (x[k] - x[k - 1]) * (t - cdf[k - 1]) / (cdf[k] - cdf[k - 1])
    return dict(lnL_max=m, ml_gamma_index=am // NA, ml_log10_A_index=am % NA, ln_bayes=m + np.log(B),
                post_log10_A=post_a, post_gamma=post_g, log10_A_ul=ulv)


def lnl_of_statics(b, pc, rows):
    """ln L [R, Ng, NA] from the plan's statics (C, V, lambda, ldet) in numpy: the eigen form the kernels evaluate."""
    nc = pc["nc"]
    a2 = pc["a2"]
    Q = np.zeros((rows.shape[0], len(pc["gamma"]), len(a2)))
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        X = rows[:, s:s + n] @ pc["C"][s:s + n, :nc]                        # [R, nc]
        y = np.einsum("gji,ri->rgj", pc["V"][i][:, :nc, :nc], X)           # [R, Ng, nc]
        w = a2[None, :, None] / (1.0 + a2[None, :, None] * pc["eig"][i][:, None, :])   # [Ng, NA, nc]
        Q += np.einsum("rgj,gkj->rgk", y * y, w)
    return 0.5 * Q - 0.5 * pc["ldet"][None]
