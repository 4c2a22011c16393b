"""TEST INFRASTRUCTURE ONLY -- dense oracle of the sine-Gaussian burst search (``PulsarBatch.set_burst_statistic``).

Builds on the dense optimal-statistic oracle (tests/os_oracle.py): every pulsar's noise covariance P_a as an explicit
n_a x n_a matrix (with the optional common process on its own k / Tspan basis) and P_a^{-1} W, or G (G^T P_a G)^{-1} G^T W
with G the SVD null space of the timing model, by dense solves.  The wavelets W [n_a, 2J] come from the TOAs' MJDs
(t = MJD 86400) and the template table, each on the span of TOAs with |t - t0| <= 6 tau.  ``emulate`` restates the
device's factored arithmetic (N^-1 r per ECORR run, z, W^T N^-1 r - H^T z) in numpy from the plan.  Nothing here
imports the product's statics code."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def windows(b, i, templates):
    """[J, 2] (lo, hi): the span of pulsar ``i``'s TOAs (engine order) from the first to the last with |t - t0| <= 6 tau."""
    t = np.asarray(b.psrs[i].toas.get_mjds().value, dtype=np.float64)[b.order[i]] * 86400
    out = np.zeros((len(templates), 2), dtype=np.int64)
    for j, (t0, f0, Q) in enumerate(templates):
        tau = Q / (2 * np.pi * f0)
        ins = np.flatnonzero(np.abs(t - t0 * 86400) <= 6 * tau)
        if ins.size:
            out[j] = ins[0], ins[-1] + 1
    return out


def wavelets(b, i, templates):
    """[n_a, 2J] W (column 2 j + c, c = 0 cos, 1 sin) of pulsar ``i`` in engine order, zero outside each window."""
    t = np.asarray(b.psrs[i].toas.get_mjds().value, dtype=np.float64)[b.order[i]] * 86400
    W = np.zeros((len(t), 2 * len(templates)))
    for j, ((t0, f0, Q), (lo, hi)) in enumerate(zip(templates, windows(b, i, templates))):
        x = t[lo:hi] - t0 * 86400
        g = np.exp(-(x * 2 * np.pi * f0 / Q) ** 2)
        W[lo:hi, 2 * j], W[lo:hi, 2 * j + 1] = g * np.cos(2 * np.pi * f0 * x), g * np.sin(2 * np.pi * f0 * x)
    return W


def statics(b, templates, log10_A_common=None, gamma_common=13 / 3, components_common=14, models=None):
    """Dense statics per pulsar: W, C = P_a^{-1} W, M [J, 2, 2] = W^T C, the trace of W^T N_white^-1 W and seen."""
    Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    out = dict(W=[], C=[], M=[], seen=[])
    for i in range(b.n_psr):
        W = wavelets(b, i, templates)
        pc = None if log10_A_common is None else 10 ** (2 * log10_A_common) * OO.phi_tilde(components_common, gamma_common,
                                                                                         Tspan)
        Pa = OO.dense_covariance(b, i, OO.gw_basis(b.t_tdb[i], components_common, Tspan), pc)
        Ca = OO.c_matrix(Pa, W, None if models is None else models[i])
        M = np.einsum("nji,njk->jik", W.reshape(len(W), -1, 2), Ca.reshape(len(W), -1, 2))
        M = 0.5 * (M + M.transpose(0, 2, 1))
        w1, w2 = b._white[i]
        tr = (W * W / (w1**2 + w2**2)[:, None]).reshape(len(W), -1, 2).sum(axis=(0, 2))
        out["W"].append(W)
        out["C"].append(Ca)
        out["M"].append(M)
        out["seen"].append(np.linalg.eigvalsh(M)[:, 0] > 1e-12 * tr)
    out["M"], out["seen"] = np.stack(out["M"]), np.stack(out["seen"])
    return out


def dense_n(b, S, rows):
    """W^T P_a^{-1} r [R, P, J, 2] of engine-order rows [R, ld]."""
    return np.stack([(rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ S["C"][i]).reshape(len(rows), -1, 2)
                     for i in range(b.n_psr)], axis=1)


def emulate(b, pb, rows, dtype=np.float64):
    """The device's arithmetic in numpy (``dtype``) from ``plan()["burst"]``: y = N^-1 r per ECORR run, z from the z
    columns, N = W^T y - H^T z with W regenerated from the template table on each window.  Returns N [R, P, J, 2] and
    the whitened X^ = L^-1 N (0 at unseen cells)."""
    from pta_replicator_b200.engine import fp_whitened_basis
    rows = np.asarray(rows, dtype=dtype)
    R, J = len(rows), pb["n_tmpl"]
    y = np.zeros_like(rows)
    for s0, ln, c in zip(pb["run_start"], pb["run_len"], pb["run_coef"]):
        x = rows[:, s0:s0 + ln]
        di = np.asarray(pb["dinv"][s0:s0 + ln], dtype=dtype)
        y[:, s0:s0 + ln] = (x - dtype(c) * (x * di).sum(axis=1, keepdims=True)) * di
    t0, itau, f2 = (np.asarray(pb["tmpl"][:, k], dtype=np.float64) for k in range(3))
    N = np.zeros((R, b.n_psr, J, 2), dtype=dtype)
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        z = rows[:, s:s + n] @ np.asarray(fp_whitened_basis(pb["z"], s, n), dtype=dtype)
        t = pb["t"][s:s + n]
        for j in range(J):
            lo, hi = pb["win"][i, j]
            x = t[lo:hi] - t0[j]
            g = np.exp(-(x * itau[j]) ** 2)
            W = np.stack([g * np.cos(np.pi * f2[j] * x), g * np.sin(np.pi * f2[j] * x)], axis=1).astype(dtype)
            N[:, i, j] = y[:, s + lo:s + hi] @ W - z @ np.asarray(pb["H"][i, j].T, dtype=dtype)
    wl = np.asarray(pb["wl"], dtype=dtype)
    X = np.stack([wl[None, ..., 0] * N[..., 0], wl[None, ..., 1] * N[..., 0] + wl[None, ..., 2] * N[..., 1]], axis=-1)
    return N, X


def coherent(pb, X, ant):
    """B [R, J, S] and b^ = M4^-1 N4 [R, J, S, 4] (index 2 pol + c) from whitened X [R, P, J, 2] by explicit 4 x 4 solves
    of M4 = sum_a e_a e_a^T (x) M_a over the seen pulsars."""
    M = pb["M"]                                                          # [P, J, 2, 2], zero when unseen
    l11, l21, l22 = (pb["Lf"].transpose(1, 0, 2)[..., k] for k in range(3))   # [P, J]
    N = np.stack([l11 * X[..., 0], l21 * X[..., 0] + l22 * X[..., 1]], axis=-1)   # L X^ = W^T P^-1 r
    R, P, J, _ = X.shape
    S = ant.shape[1]
    B, bh = np.empty((R, J, S)), np.empty((R, J, S, 4))
    for j in range(J):
        M4 = np.einsum("asp,asq,aij->spiqj", ant, ant, M[:, j]).reshape(S, 4, 4)
        N4 = np.einsum("asp,rai->rspi", ant, N[:, :, j]).reshape(R, S, 4)
        sol = np.linalg.solve(M4[None], N4[..., None])[..., 0]
        B[:, j] = 0.5 * np.sum(N4 * sol, axis=-1)
        bh[:, j] = sol
    return B, bh
