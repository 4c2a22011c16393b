"""TEST INFRASTRUCTURE ONLY -- dense oracle of the optimal statistic (``PulsarBatch.set_optimal_statistic``).

An independent restatement for small batches: it builds every pulsar's noise covariance P_a as an explicit n_a x n_a
matrix from the recipe the batch holds (white variances, ECORR buckets, red-noise frequencies and priors), takes the
null space G of the timing design matrix from an SVD, and computes C_a = G (G^T P_a G)^{-1} G^T F_gw,a with dense
solves -- no Woodbury, no Sherman-Morrison.  The Hellings-Downs template is the closed form 1.5 x ln x - x / 4 + 1/2,
x = (1 - cos zeta) / 2.  ``expected_a2`` gives the exact E[A2] of an injected GWB from the injection covariance.
Nothing here imports the product's statics code."""
from __future__ import annotations

import numpy as np

YEAR = 365.25 * 24 * 3600


def gw_basis(t, K, Tspan):
    """[n, 2K]: (sin, cos)(2 pi k t / Tspan), k = 1..K."""
    f = np.arange(1, K + 1) / Tspan
    arg = 2 * np.pi * np.outer(t, f)
    return np.stack([np.sin(arg), np.cos(arg)], axis=2).reshape(len(t), 2 * K)


def phi_tilde(K, gamma, Tspan):
    f = np.repeat(np.arange(1, K + 1) / Tspan, 2)
    return (f * YEAR) ** (-gamma) / (12 * np.pi**2 * Tspan) * YEAR**3


def dense_covariance(b, i, Fgw=None, phi_common=None):
    """P_a in engine order from the batch's recipe (white + ECORR + red noise + optional common process)."""
    w1, w2 = b._white[i]
    P = np.diag(w1**2 + w2**2)
    if b._ecorr is not None and b._ecorr[i] is not None:
        bucket, e = b._ecorr[i]
        P = P + (np.asarray(e)[bucket] ** 2)[:, None] * (bucket[:, None] == bucket[None, :])
    if b._red is not None and b._red["f"][i] is not None:
        f = np.asarray(b._red["f"][i])
        arg = 2 * np.pi * np.outer(b.t_tdb[i], f)
        Fr = np.empty((len(arg), 2 * len(f)))
        Fr[:, 0::2], Fr[:, 1::2] = np.sin(arg), np.cos(arg)
        P = P + (Fr * np.asarray(b._red["scale"][i]) ** 2) @ Fr.T
    if phi_common is not None:
        P = P + (Fgw * phi_common) @ Fgw.T
    return P


def c_matrix(P, F, M=None):
    """P^{-1} F, or with a timing model M: G (G^T P G)^{-1} G^T F, G = null space of M^T (SVD)."""
    if M is None:
        return np.linalg.solve(P, F)
    U, s, _ = np.linalg.svd(M, full_matrices=True)
    G = U[:, int(np.sum(s > 1e-10 * s[0])):]
    return G @ np.linalg.solve(G.T @ P @ G, G.T @ F)


def hd_closed_form(b):
    """Hellings-Downs, Gamma_aa = 1, from the pulsar positions (RAJ [h], DECJ [deg])."""
    ra = np.array([p.loc["RAJ"] * np.pi / 12 for p in b.psrs])
    dec = np.array([p.loc["DECJ"] * np.pi / 180 for p in b.psrs])
    u = np.stack([np.cos(dec) * np.cos(ra), np.cos(dec) * np.sin(ra), np.sin(dec)], axis=1)
    c = np.clip(u @ u.T, -1, 1)
    x = (1 - c) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        h = 1.5 * x * np.log(x) - x / 4 + 0.5
    np.fill_diagonal(h, 1.0)
    return h, c


def statics(b, K=14, gamma=13 / 3, Tspan=None, log10_A_common=None, models=None, templates=("hd", "monopole", "dipole")):
    """Dense statics: dict(C [per pulsar n_a x 2K], Z, t [P, P], W [n_orf, n_pairs], D, F, Finv, phi, pairs)."""
    P = b.n_psr
    if Tspan is None:
        Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    phi = phi_tilde(K, gamma, Tspan)
    Cs, Z = [], []
    for i in range(P):
        F = gw_basis(b.t_tdb[i], K, Tspan)
        pc = None if log10_A_common is None else 10 ** (2 * log10_A_common) * phi
        Pa = dense_covariance(b, i, F, pc)
        Ca = c_matrix(Pa, F, None if models is None else models[i])
        Cs.append(Ca)
        Z.append(F.T @ Ca)
    t = np.array([[np.trace(Z[a] @ np.diag(phi) @ Z[c] @ np.diag(phi)) for c in range(P)] for a in range(P)])
    pa, pb = np.triu_indices(P, 1)
    h, cz = hd_closed_form(b)
    mats = {"hd": h, "monopole": np.ones((P, P)), "dipole": cz}
    W = np.stack([mats[o][pa, pb] if isinstance(o, str) else np.asarray(o)[pa, pb] for o in templates])
    tab = t[pa, pb]
    F_ = (W * tab) @ W.T
    return dict(C=Cs, Z=np.stack(Z), t=t, W=W, D=(W * W) @ tab, F=F_, Finv=np.linalg.inv(F_), phi=phi, pairs=(pa, pb))


def os_of_rows(b, S, rows):
    """rho [R, n_pairs], A2, snr, A2_mc [R, n_orf] of engine-order rows [R, ld] from dense statics ``S``."""
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ S["C"][i] for i in range(b.n_psr)], axis=1)
    pa, pb = S["pairs"]
    d = np.einsum("rpj,rpj->rp", X[:, pa] * S["phi"], X[:, pb])
    tab = S["t"][pa, pb]
    bo = d @ S["W"].T
    return dict(rho=d / tab, A2=bo / S["D"], snr=bo / np.sqrt(S["D"]), A2_mc=bo @ S["Finv"].T)


def gwb_synthesis_matrix(g):
    """The GWB injection's grid synthesis T [npts, 2(Nf-2)] (pruned inverse DFT times sqrt(C)), so that the grid of
    pulsar p is T z_p with z ~ N(0, 1) mixed across pulsars by the ORF: cov(grid_a, grid_b) = ORF_ab T T^T."""
    Nf, npts, dt = g["Nf"], g["npts"], g["dt"]
    N = 2 * Nf - 2
    kk = np.arange(1, Nf - 1)
    nn = np.arange(npts) + 10
    ang = 2 * np.pi * ((kk[None, :] * nn[:, None]) % N) / N
    s = (2.0 / (N * dt)) * np.sqrt(g["C"][1:Nf - 1])
    T = np.zeros((npts, 2 * (Nf - 2)))
    T[:, 0::2] = np.cos(ang) * s
    T[:, 1::2] = -np.sin(ang) * s
    return T


def interpolation_matrix(ut, x):
    """Linear interpolation weights W [len(x), len(ut)] on the grid ut."""
    j = np.clip(np.searchsorted(ut, x, side="right") - 1, 0, len(ut) - 2)
    w = (x - ut[j]) / (ut[j + 1] - ut[j])
    W = np.zeros((len(x), len(ut)))
    W[np.arange(len(x)), j] = 1 - w
    W[np.arange(len(x)), j + 1] = w
    return W


def expected_a2(b, S):
    """Exact E[A2_o] of the batch's injected GWB: E[x_a . x_b] = ORF_ab tr(phi~ U_a^T U_b), U_a = T^T W_a^T C_a."""
    g = b._gwb
    T = gwb_synthesis_matrix(g)
    U = [T.T @ (interpolation_matrix(g["ut"], b.mjd[i] * 86400.0).T @ S["C"][i]) for i in range(b.n_psr)]
    pa, pb = S["pairs"]
    e = np.array([g["ORF"][a, c] * np.sum(S["phi"] * np.einsum("kj,kj->j", U[a], U[c])) for a, c in zip(pa, pb)])
    return (S["W"] @ e) / S["D"]
