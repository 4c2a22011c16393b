"""TEST INFRASTRUCTURE ONLY -- dense oracle of the per-frequency optimal statistic (``PulsarBatch.set_os_per_frequency``).

Built on the dense statics of tests/os_oracle.py (explicit P_a, null-space solves), nothing from the product's statics
code.  With X_a = C_a^T r_a the unscaled projection of pulsar a, Z_a = F_gw,a^T C_a and Z_a[k] its 2 x 2 diagonal
block at f_k = k / Tspan:
    t_qk = tr(Z_a[k] Z_b[k])  (explicit traces),  D_ok = sum_q (Gamma^o_q)^2 t_qk,  F_k = W diag(t_k) W^T;
    d_qk = X_a,2k X_b,2k + X_a,2k+1 X_b,2k+1,  phi_ok = sum_q Gamma^o_q d_qk / D_ok,  phi_mc_k = F_k^{-1} b_k.
``expected_pf_phi`` gives the exact E[phi_ok] of the batch's injected GWB: E[X_a,j X_b,j] = ORF_ab (U_a^T U_b)_jj with
U_a = T^T W_a^T C_a (T the injection's grid synthesis, W_a the interpolation to the TOAs), the per-column form of
``os_oracle.expected_a2`` without the phi~ weights."""
from __future__ import annotations

import numpy as np

from tests import os_oracle as OO


def pf_statics(b, S):
    """dict(t [K, n_pairs], D [n_orf, K], F [K, n_orf, n_orf], Finv [K, n_orf, n_orf], K) of dense statics ``S``."""
    Z, W = S["Z"], S["W"]
    K = Z.shape[1] // 2
    pa, pb = S["pairs"]
    t = np.empty((K, len(pa)))
    for k in range(K):
        s = slice(2 * k, 2 * k + 2)
        for q, (a, c) in enumerate(zip(pa, pb)):
            t[k, q] = np.trace(Z[a][s, s] @ Z[c][s, s])
    F = np.stack([(W * t[k]) @ W.T for k in range(K)])
    return dict(K=K, t=t, D=(W * W) @ t.T, F=F, Finv=np.linalg.inv(F))


def projections(b, S, rows):
    """X [R, P, 2K]: the unscaled projections of engine-order rows [R, ld]."""
    return np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ S["C"][i] for i in range(b.n_psr)], axis=1)


def pf_of_rows(b, S, rows, T=None):
    """rho [R, K, n_pairs], phi, snr, phi_mc [R, n_orf, K] of rows [R, ld] (``T``: ``pf_statics``, computed when None)."""
    T = pf_statics(b, S) if T is None else T
    X = projections(b, S, rows)
    R, K = len(rows), T["K"]
    pa, pb = S["pairs"]
    d = (X[:, pa] * X[:, pb]).reshape(R, len(pa), K, 2).sum(axis=3).transpose(0, 2, 1)    # [R, K, n_pairs]
    bo = np.einsum("oq,rkq->rok", S["W"], d)
    return dict(rho=d / T["t"], phi=bo / T["D"], snr=bo / np.sqrt(T["D"]),
                phi_mc=np.einsum("kop,rpk->rok", T["Finv"], bo))


def expected_pf_phi(b, S, T=None):
    """Exact E[phi_ok] [n_orf, K] of the batch's injected GWB (``set_gwb``)."""
    T = pf_statics(b, S) if T is None else T
    g = b._gwb
    Tg = OO.gwb_synthesis_matrix(g)
    U = [Tg.T @ (OO.interpolation_matrix(g["ut"], b.mjd[i] * 86400.0).T @ S["C"][i]) for i in range(b.n_psr)]
    pa, pb = S["pairs"]
    e = np.array([g["ORF"][a, c] * np.einsum("kj,kj->j", U[a], U[c]) for a, c in zip(pa, pb)])    # [n_pairs, 2K]
    ed = e.reshape(len(pa), T["K"], 2).sum(axis=2).T                                              # [K, n_pairs]
    return (S["W"] @ ed.T) / T["D"]
