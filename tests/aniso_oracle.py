"""TEST INFRASTRUCTURE ONLY -- dense oracle of the anisotropy statistics of the optimal statistic
(``PulsarBatch.set_os_anisotropy``).

Built on the dense optimal-statistic oracle (tests/os_oracle.py): rho_q = d_q / t_q with weights t_q (sigma_q^2 = 1 / t_q).
  * Spherical harmonics: c^ is the weighted least-squares fit of rho by the templates B_lm[a, b] (``np.linalg.lstsq`` of
    sqrt(t) rho ~ sqrt(t) T^T c, not the F^{-1} fold of the product), and the anisotropy chi^2 gain is the difference
    of the isotropic (l = 0 only) and the full fits' chi^2 minima.  The templates are ``orf.correlated_basis``, pinned
    to the reference by tests/test_oracle_pinning.py.
  * Radiometer: the antenna patterns come from the polarisation tensors e+ = m m - n n and ex = m n + n m of the
    ``add_cgw`` source frame, F^A = 1/2 p^i p^j e^A_ij / (1 + Omega . p), not from ``engine.antenna_patterns``;
    T_k,q = 3 / (2 S) sum_A F^A_a F^A_b and S/N_k = sum_q T_k,q d_q / sqrt(sum_q T_k,q^2 t_q).
  * ``expected_pair_means``: the exact E[d_q] of the batch's injected GWB, E[x_a . x_b] = ORF_ab tr(phi~ U_a^T U_b)
    with U_a = T^T W_a^T C_a (the per-pair vector of ``os_oracle.expected_a2``, restated)."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def pulsar_units(b):
    """[P, 3] unit vectors to the pulsars (RAJ [h], DECJ [deg])."""
    ra = np.array([p.loc["RAJ"] * np.pi / 12 for p in b.psrs])
    dec = np.array([p.loc["DECJ"] * np.pi / 180 for p in b.psrs])
    return np.stack([np.cos(dec) * np.cos(ra), np.cos(dec) * np.sin(ra), np.sin(dec)], axis=1)


def sph_templates(b, lmax, pairs):
    """[n_lm, n_pairs] B_lm[a, b], (l, m = -l..l)."""
    from pta_replicator_b200 import orf
    ra = np.array([p.loc["RAJ"] * np.pi / 12 for p in b.psrs])
    dec = np.array([p.loc["DECJ"] * np.pi / 180 for p in b.psrs])
    B = orf.correlated_basis(np.stack([ra, np.pi / 2 - dec], axis=1), lmax)
    return np.stack([m[pairs[0], pairs[1]] for m in B])


def antenna_tensor(b, sky):
    """[P, S, 2] (F+, Fx) from the polarisation tensors at sky points (gwtheta, gwphi)."""
    th, ph = sky[:, 0], sky[:, 1]
    m = np.stack([np.sin(ph), -np.cos(ph), np.zeros_like(ph)], axis=1)
    n = np.stack([-np.cos(th) * np.cos(ph), -np.cos(th) * np.sin(ph), np.sin(th)], axis=1)
    om = -np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], axis=1)
    ep = np.einsum("si,sj->sij", m, m) - np.einsum("si,sj->sij", n, n)
    ex = np.einsum("si,sj->sij", m, n) + np.einsum("si,sj->sij", n, m)
    p = pulsar_units(b)
    den = 1.0 + p @ om.T                                                      # [P, S]
    fp = 0.5 * np.einsum("ai,aj,sij->as", p, p, ep) / den
    fx = 0.5 * np.einsum("ai,aj,sij->as", p, p, ex) / den
    return np.stack([fp, fx], axis=2)


def radio_templates(b, sky, pairs):
    ant = antenna_tensor(b, sky)
    return 1.5 / len(sky) * np.einsum("qkp,qkp->kq", ant[pairs[0]], ant[pairs[1]])


def pair_correlations(b, S, rows):
    """d [R, n_pairs] and t [n_pairs] of engine-order rows from dense statics ``S`` (os_oracle.statics)."""
    pa, pb = S["pairs"]
    t = S["t"][pa, pb]
    return OO.os_of_rows(b, S, rows)["rho"] * t, t


def sph_fit(d, t, T):
    """c^ [R, n_lm] and the anisotropy chi^2 gain [R] by weighted least squares of rho = d / t."""
    w = np.sqrt(t)
    rho = d / t
    A = (T * w).T                                                             # [n_pairs, n_lm]
    c = np.stack([np.linalg.lstsq(A, w * r, rcond=None)[0] for r in rho])
    full = np.sum((w * (rho - c @ T)) ** 2, axis=1)
    c0 = (rho * t) @ T[0] / (T[0] ** 2 @ t)
    iso = np.sum((w * (rho - c0[:, None] * T[0])) ** 2, axis=1)
    return c, iso - full


def radiometer(d, t, Tr):
    """S/N [R, S] and sigma [S]."""
    Fkk = (Tr * Tr) @ t
    return d @ Tr.T / np.sqrt(Fkk), 1.0 / np.sqrt(Fkk)


def expected_pair_means(b, S):
    """Exact E[d_q] [n_pairs] of the batch's injected GWB (``set_gwb``)."""
    g = b._gwb
    T = OO.gwb_synthesis_matrix(g)
    U = [T.T @ (OO.interpolation_matrix(g["ut"], b.mjd[i] * 86400.0).T @ S["C"][i]) for i in range(b.n_psr)]
    pa, pb = S["pairs"]
    return np.array([g["ORF"][a, c] * np.sum(S["phi"] * np.einsum("kj,kj->j", U[a], U[c])) for a, c in zip(pa, pb)])
