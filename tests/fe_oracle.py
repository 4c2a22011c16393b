"""TEST INFRASTRUCTURE ONLY -- dense oracle of the Fe-statistic (``PulsarBatch.set_fe_statistic``).

Builds on the dense Fp oracle (tests/fp_oracle.py: explicit P_a, C_a by dense solves, numpy Cholesky L_a(f) of M_a(f),
the whitened basis C~_a(f)).  Per cell (f, s) it forms the explicit 2P x 4 design matrix of a continuous wave in the
whitened amplitudes,
    H(f, s) = [L_a(f)^T E_a(s)]_a,   E_a(s) = [F+_a(s) I_2, Fx_a(s) I_2]   (2 x 4),
so that X^ = H b + noise for the 4 amplitudes b = (A+ sin, A+ cos, Ax sin, Ax cos), and evaluates
    Fe = 1/2 (H^T X^)^T (H^T H)^{-1} (H^T X^)
by a numpy solve.  The antenna patterns are the ``add_cgw`` formula evaluated pulsar by pulsar with ``np.dot`` from the
pulsars' RAJ / DECJ, (0, 0) where 1 + Omega.p <= 1e-12.  Nothing here imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import fp_oracle as FO
from tests import os_oracle as OO


def antenna(b, sky):
    """[P, S, 2] (F+, Fx) of every pulsar of ``b`` for sources at ``sky`` [S, 2] (gwtheta, gwphi)."""
    sky = np.asarray(sky, dtype=float)
    out = np.zeros((b.n_psr, len(sky), 2))
    for i, p in enumerate(b.psrs):
        ptheta = np.pi / 2 - p.loc["DECJ"] * np.pi / 180
        pphi = p.loc["RAJ"] * np.pi / 12
        phat = np.array([np.sin(ptheta) * np.cos(pphi), np.sin(ptheta) * np.sin(pphi), np.cos(ptheta)])
        for s, (th, ph) in enumerate(sky):
            m = np.array([np.sin(ph), -np.cos(ph), 0.0])
            n = np.array([-np.cos(th) * np.cos(ph), -np.cos(th) * np.sin(ph), np.sin(th)])
            om = np.array([-np.sin(th) * np.cos(ph), -np.sin(th) * np.sin(ph), -np.cos(th)])
            den = 1 + np.dot(om, phat)
            if den > 1e-12:
                out[i, s] = 0.5 * (np.dot(m, phat) ** 2 - np.dot(n, phat) ** 2) / den, np.dot(m, phat) * np.dot(n, phat) / den
    return out


def design(S, ant, f, s):
    """H(f, s) [2P, 4] of the dense Fp statics ``S`` (tests/fp_oracle.py) and antenna patterns ``ant``."""
    P = len(S["L"])
    H = np.zeros((2 * P, 4))
    for a in range(P):
        E = np.hstack([ant[a, s, 0] * np.eye(2), ant[a, s, 1] * np.eye(2)])
        H[2 * a:2 * a + 2] = S["L"][a][f].T @ E
    return H


def fe_of_amps(S, ant, X):
    """Fe [R, Nf, S] of whitened amplitudes X [R, P, Nf, 2]."""
    R, P, Nf, _ = X.shape
    nsky = ant.shape[1]
    out = np.empty((R, Nf, nsky))
    for f in range(Nf):
        xf = X[:, :, f, :].reshape(R, 2 * P)
        for s in range(nsky):
            H = design(S, ant, f, s)
            u = xf @ H                                                  # [R, 4] = H^T X^
            out[:, f, s] = 0.5 * np.sum(u * np.linalg.solve(H.T @ H, u.T).T, axis=1)
    return out


def fe_of_rows(b, S, ant, rows):
    """Fe [R, Nf, S] of engine-order rows [R, ld]."""
    return fe_of_amps(S, ant, FO.amps_of_rows(b, S, rows))


def signal_power(b, S, signal_row, models=None):
    """<s|s> = sum_a s_a^T P_a^{-1} s_a of a deterministic signal (one engine-order row) by dense solves, with the timing
    model ``models[a]`` marginalised as in tests/os_oracle.py's ``c_matrix``."""
    row = np.asarray(signal_row)
    tot = 0.0
    for i in range(b.n_psr):
        sa = row[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]]
        tot += float(sa @ OO.c_matrix(S["P"][i], sa[:, None], None if models is None else models[i])[:, 0])
    return tot
