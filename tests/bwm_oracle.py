"""TEST INFRASTRUCTURE ONLY -- dense oracle of the burst-with-memory search (``PulsarBatch.set_bwm_statistic``).

Builds on the dense optimal-statistic and Fp oracles (tests/os_oracle.py, tests/fp_oracle.py): every pulsar's noise
covariance P_a as an explicit n_a x n_a matrix (with the optional common process on its own k / Tspan basis) and
C_a = P_a^{-1} u, or G (G^T P_a G)^{-1} G^T u with G the SVD null space of the timing model, by dense solves.  The ramps
u [n_a, T] come from the TOAs' MJDs (t = MJD 86400, u = t - t0 for t >= t0).  Per cell (t0, s) it forms the explicit
P x 2 design matrix of a memory burst in the whitened amplitudes, H[a] = sqrt(m_a(t0)) e_a(s), so that
X^ = H b + noise for b = h (cos 2 psi, sin 2 psi), and evaluates B = 1/2 (H^T X^)^T (H^T H)^{-1} (H^T X^) and
b^ = (H^T H)^{-1} H^T X^ by numpy solves.  Nothing here imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def ramps(b, i, t0_mjd):
    """[n_a, T] u(t) = t - t0 (t >= t0) else 0 of pulsar ``i`` in engine order, t = MJD 86400 from the TOA table."""
    mjd = np.asarray(b.psrs[i].toas.get_mjds().value, dtype=np.float64)[b.order[i]]
    t = mjd * 86400
    ts = np.asarray(t0_mjd, dtype=float) * 86400
    return np.where(t[:, None] < ts[None, :], 0.0, t[:, None] - ts[None, :])


def statics(b, t0_mjd, log10_A_common=None, gamma_common=13 / 3, components_common=14, models=None):
    """Dense statics: P (per pulsar), m [P, T], seen [P, T], Ct (per pulsar [n_a, T], zero for unseen epochs)."""
    Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    T = len(t0_mjd)
    out = dict(P=[], Ct=[], m=np.zeros((b.n_psr, T)), seen=np.zeros((b.n_psr, T), dtype=bool))
    for i in range(b.n_psr):
        u = ramps(b, i, t0_mjd)
        pc = None if log10_A_common is None else 10 ** (2 * log10_A_common) * OO.phi_tilde(components_common, gamma_common,
                                                                                         Tspan)
        Pa = OO.dense_covariance(b, i, OO.gw_basis(b.t_tdb[i], components_common, Tspan), pc)
        Ca = OO.c_matrix(Pa, u, None if models is None else models[i])
        m = np.sum(u * Ca, axis=0)
        w1, w2 = b._white[i]
        seen = m > 1e-12 * np.sum(u * u / (w1**2 + w2**2)[:, None], axis=0)
        Ct = np.zeros_like(Ca)
        Ct[:, seen] = Ca[:, seen] / np.sqrt(m[seen])
        out["P"].append(Pa)
        out["Ct"].append(Ct)
        out["m"][i] = np.where(seen, m, 0.0)
        out["seen"][i] = seen
    return out


def amps_of_rows(b, S, rows):
    """X^ [R, P, T] = C~_a^T r_a of engine-order rows [R, ld]."""
    return np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ S["Ct"][i] for i in range(b.n_psr)], axis=1)


def design(S, ant, t, s):
    """H(t0, s) [P, 2]: row a = sqrt(m_a(t0)) e_a(s)."""
    return np.sqrt(S["m"][:, t])[:, None] * ant[:, s, :]


def bwm_of_amps(S, ant, X):
    """B [R, T, S] and b^ [R, T, S, 2] of whitened amplitudes X [R, P, T]."""
    R, P, T = X.shape
    nsky = ant.shape[1]
    B = np.empty((R, T, nsky))
    bh = np.empty((R, T, nsky, 2))
    for t in range(T):
        for s in range(nsky):
            H = design(S, ant, t, s)
            u = X[:, :, t] @ H                                              # [R, 2] = H^T X^
            bb = np.linalg.solve(H.T @ H, u.T).T
            B[:, t, s] = 0.5 * np.sum(u * bb, axis=1)
            bh[:, t, s] = bb
    return B, bh


def bwm_of_rows(b, S, ant, rows):
    """B [R, T, S] of engine-order rows [R, ld]."""
    return bwm_of_amps(S, ant, amps_of_rows(b, S, rows))[0]
