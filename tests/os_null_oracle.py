"""TEST INFRASTRUCTURE ONLY -- dense oracle of the optimal statistic's null distributions (``PulsarBatch.set_os_null``).

Built on tests/os_oracle.py (explicit P_a, SVD null space of the timing model, dense solves).  Phase shifts are taken
literally: every pulsar's GW basis is (sin, cos)(2 pi f_k t + phi_a,k), and C, Z, t and the normalisers are recomputed
from scratch with that basis.  Sky scrambles use the closed-form Hellings-Downs curve and cos zeta at given positions.
The dicts have the keys of ``os_oracle.statics``, so ``os_oracle.os_of_rows`` and ``os_oracle.expected_a2`` apply.
Nothing here imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def shifted_gw_basis(t, K, Tspan, phases):
    """[n, 2K]: (sin, cos)(2 pi k t / Tspan + phases[k - 1]), k = 1..K."""
    f = np.arange(1, K + 1) / Tspan
    arg = 2 * np.pi * np.outer(t, f) + np.asarray(phases, dtype=float)[None, :]
    return np.stack([np.sin(arg), np.cos(arg)], axis=2).reshape(len(t), 2 * K)


def templates_at(radec):
    """(Hellings-Downs with Gamma_aa = 1, cos zeta) [P, P] for pulsars at ``radec`` [P, 2] = (RA, DEC) in radians."""
    ra, dec = np.asarray(radec, dtype=float)[:, 0], np.asarray(radec, dtype=float)[:, 1]
    u = np.stack([np.cos(dec) * np.cos(ra), np.cos(dec) * np.sin(ra), np.sin(dec)], axis=1)
    c = np.clip(u @ u.T, -1, 1)
    x = (1 - c) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        h = 1.5 * x * np.log(x) - x / 4 + 0.5
    np.fill_diagonal(h, 1.0)
    return h, c


def phase_shifted_statics(b, phases, K=14, gamma=13 / 3, Tspan=None, log10_A_common=None, models=None,
                          templates=("hd", "monopole", "dipole")):
    """``os_oracle.statics`` with every pulsar's GW basis phase-shifted by ``phases`` [P, K]."""
    P = b.n_psr
    if Tspan is None:
        Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    phi = OO.phi_tilde(K, gamma, Tspan)
    Cs, Z = [], []
    for i in range(P):
        F = shifted_gw_basis(b.t_tdb[i], K, Tspan, phases[i])
        pc = None if log10_A_common is None else 10 ** (2 * log10_A_common) * phi
        Ca = OO.c_matrix(OO.dense_covariance(b, i, F, pc), F, None if models is None else models[i])
        Cs.append(Ca)
        Z.append(F.T @ Ca)
    t = np.array([[np.trace(Z[a] @ np.diag(phi) @ Z[c] @ np.diag(phi)) for c in range(P)] for a in range(P)])
    pa, pb = np.triu_indices(P, 1)
    h, cz = OO.hd_closed_form(b)
    mats = {"hd": h, "monopole": np.ones((P, P)), "dipole": cz}
    W = np.stack([mats[o][pa, pb] if isinstance(o, str) else np.asarray(o)[pa, pb] for o in templates])
    tab = t[pa, pb]
    F_ = (W * tab) @ W.T
    return dict(C=Cs, Z=np.stack(Z), t=t, W=W, D=(W * W) @ tab, F=F_, Finv=np.linalg.inv(F_), phi=phi, pairs=(pa, pb))


def scrambled_statics(S, radec, template="hd"):
    """Statics ``S`` of ``os_oracle.statics`` with the single template ``template`` ("hd" or "dipole") rebuilt at the
    positions ``radec`` [P, 2]; C, Z and t are unchanged by a scramble."""
    h, cz = templates_at(radec)
    pa, pb = S["pairs"]
    W = (h if template == "hd" else cz)[pa, pb][None]
    tab = S["t"][pa, pb]
    F_ = (W * tab) @ W.T
    return dict(S, W=W, D=(W * W) @ tab, F=F_, Finv=np.linalg.inv(F_))
