"""TEST INFRASTRUCTURE ONLY -- dense oracle of the Fp-statistic (``PulsarBatch.set_fp_statistic``).

Builds on the dense optimal-statistic oracle (tests/os_oracle.py): every pulsar's noise covariance P_a as an explicit
n_a x n_a matrix (``dense_covariance``, with the optional common process on its own k / Tspan basis) and
C_a = P_a^{-1} F, or G (G^T P_a G)^{-1} G^T F with G the SVD null space of the timing model (``c_matrix``), by dense
solves.  Then per search frequency f: M_a(f) = F_f^T C_a(f), its Cholesky factor L (numpy) and the whitened basis
C~_a(f) = C_a(f) L^{-T}; the Fp-statistic of rows and the noncentrality lambda_f of a deterministic signal.  Nothing here
imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def fp_basis(t, freqs):
    """[n, 2 Nf]: (sin, cos)(2 pi f t) per search frequency."""
    arg = 2 * np.pi * np.outer(t, np.asarray(freqs, dtype=float))
    return np.stack([np.sin(arg), np.cos(arg)], axis=2).reshape(len(t), -1)


def statics(b, freqs, Tspan=None, log10_A_common=None, gamma_common=13 / 3, components_common=14, models=None):
    """Dense statics per pulsar: P (covariance), C [n, 2Nf], M [Nf, 2, 2], L [Nf, 2, 2], Ct [n, 2Nf] (C~)."""
    if Tspan is None:
        Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    Nf = len(freqs)
    out = dict(P=[], C=[], M=[], L=[], Ct=[])
    for i in range(b.n_psr):
        t = b.t_tdb[i]
        F = fp_basis(t, freqs)
        pc = None if log10_A_common is None else 10 ** (2 * log10_A_common) * OO.phi_tilde(components_common, gamma_common, Tspan)
        Pa = OO.dense_covariance(b, i, OO.gw_basis(t, components_common, Tspan), pc)
        Ca = OO.c_matrix(Pa, F, None if models is None else models[i])
        M = np.empty((Nf, 2, 2))
        L = np.empty((Nf, 2, 2))
        Ct = np.empty_like(Ca)
        for f in range(Nf):
            c = slice(2 * f, 2 * f + 2)
            m = F[:, c].T @ Ca[:, c]
            M[f] = 0.5 * (m + m.T)
            L[f] = np.linalg.cholesky(M[f])
            Ct[:, c] = np.linalg.solve(L[f], Ca[:, c].T).T
        for k, v in (("P", Pa), ("C", Ca), ("M", M), ("L", L), ("Ct", Ct)):
            out[k].append(v)
    return out


def amps_of_rows(b, S, rows):
    """X^ [R, P, Nf, 2] = C~_a^T r_a of engine-order rows [R, ld]."""
    X = [rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ S["Ct"][i] for i in range(b.n_psr)]
    return np.stack(X, axis=1).reshape(rows.shape[0], b.n_psr, -1, 2)


def fp_of_rows(b, S, rows):
    """Fp [R, Nf] = 1/2 sum_a |X^_a(f)|^2."""
    return 0.5 * np.sum(amps_of_rows(b, S, rows) ** 2, axis=(1, 3))


def noncentrality(b, S, signal_row):
    """lambda_f = sum_a |C~_a(f)^T s_a|^2 of a deterministic signal (one engine-order row): 2 Fp ~ chi^2_2P(lambda_f)."""
    return 2.0 * fp_of_rows(b, S, np.asarray(signal_row)[None, :])[0]
