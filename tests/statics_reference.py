"""TEST INFRASTRUCTURE ONLY -- extended-precision dense reference of the statistics' host statics (``plan()["os"]``,
``["os_aniso"]``, ``["fp"]``, ``["fe"]``, ``["curn"]``, ``["hd"]``) and the edge recipes they are tested at.  numpy
and mpmath only; nothing here imports the product's statics code.

The reference restates the definitions, not the product's algorithms (Woodbury over N, Sherman-Morrison per ECORR
bucket, unit-diagonal scaling, eigen forms, Cholesky whitening):

  * Tier 1, per pulsar, n_a x n_a in ``np.longdouble``.  P_a is formed from the recipe's fp64 parameters (white
    variances w1^2 + w2^2, ECORR buckets and values, red-noise frequencies and sqrt-priors, the optional common
    process), every operation after reading them in long double.  The sin / cos basis values are fp64 inputs,
    evaluated with the expression the product uses, so that both sides start from the same numbers.  P_a is factored
    by a long-double Cholesky (a column loop), every solve takes two steps of iterative refinement, and the timing
    model enters in the constrained form
        C = P^-1 F - P^-1 M (M^T P^-1 M)^-1 M^T P^-1 F
    with M the design matrix rebuilt from the recipe's columns (neither a null space nor Woodbury).  Tier 1 gives
    C_a, Z_a = F^T C_a and X_a = C_a^T r.
  * Tier 2, the small systems, in mpmath at ``DPS`` digits from the tier-1 values: CURN's 2K x 2K I + A^2 Zh per grid
    point (ln L = 1/2 y^T (I + M)^-1 y - 1/2 ln det(I + M)), HD's stacked N x N system (N = P 2K; Gamma = E mu E^T in
    mpmath), the optimal statistic's pair sums t_ab and template Fisher matrix, Fp's 2 x 2 M_a(f), Fe's 4 x 4 M4(f, s),
    the anisotropy Fisher matrix, its Schur complement and the radiometer's F_kk.  Antenna patterns are evaluated in
    mpmath from the fp64 angles.

Outputs are the definitions applied to given rows; the kernels' layouts play no part.  ``woodbury_cond`` reports
kappa of the unit-diagonal Woodbury matrix S = Phi^-1 + T^T N^-1 T of a pulsar (the system the product solves), which
the tests scale their tolerance by where a recipe is ill-conditioned.  ``self_check`` runs tier 1 entirely in mpmath
on the smallest recipe and returns the long-double path's worst relative difference.

The second half builds the edge recipes (``recipes()``): named ``Edge`` objects, each a ``plan_only`` batch plus what
the reference reads besides the batch's noise recipe (timing-model columns and the statistics' settings)."""
from __future__ import annotations

import math

import mpmath as mp
import numpy as np

from tests import reduction_reference as RR

LD = np.longdouble
LONG = RR.LONG
DPS = 45
YEAR = 365.25 * 24 * 3600          # const.YEAR_IN_SEC, the year of the set_red power law
FE_POLE_TOL = 1e-12                # 1 + Omega . p at or below this: the pattern is 0/0 and set to (0, 0)


# ------------------------------------------------------------------ tier 1: long double
def basis(t, freqs):
    """[n, 2 Nf] fp64 (sin, cos)(2 pi f t) column pairs: the product's expression, so both sides share the inputs."""
    arg = (2 * np.pi * t)[:, None] * np.asarray(freqs, dtype=float)[None, :]
    out = np.empty((len(t), 2 * arg.shape[1]))
    out[:, 0::2], out[:, 1::2] = np.sin(arg), np.cos(arg)
    return out


def array_tspan(b, Tspan=None):
    return float(Tspan) if Tspan is not None else float(max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb))


def ld_phi(freqs, gamma, Tspan, log10_A=None):
    """The set_red power-law prior per (sin, cos) column in long double (A = 1 without ``log10_A``)."""
    ff = np.repeat(np.asarray(freqs, dtype=float), 2).astype(LD)
    y = LD(YEAR)
    p = (ff * y) ** (-LD(gamma)) / (12 * LD(math.pi) ** 2 * LD(Tspan)) * y ** 3
    return p if log10_A is None else p * LD(10) ** (2 * LD(log10_A))


def covariance(b, i, common=None, own_red=True):
    """P_a [n, n] (long double): white + ECORR + red noise (left out with ``own_red`` False) + every chromatic process
    (w w^T) ⊙ (F_s phi_s F_s^T) (+ common: (basis [n, m] fp64, prior [m] long double))."""
    w1, w2 = (np.asarray(v, dtype=float).astype(LD) for v in b._white[i])
    P = np.diag(w1 * w1 + w2 * w2)
    if b._ecorr is not None and b._ecorr[i] is not None:
        bucket, e = b._ecorr[i]
        e2 = np.asarray(e, dtype=float).astype(LD)[bucket] ** 2
        P = P + np.where(bucket[:, None] == bucket[None, :], e2[:, None], LD(0))
    if own_red and b._red is not None and b._red["f"][i] is not None:
        Fr = basis(b.t_tdb[i], b._red["f"][i]).astype(LD)
        P = P + (Fr * np.asarray(b._red["scale"][i], dtype=float).astype(LD) ** 2) @ Fr.T
    for Fw, phi in chrom_blocks(b, i):
        P = P + (Fw * phi) @ Fw.T
    if common is not None:
        Fc = common[0].astype(LD)
        P = P + (Fc * common[1]) @ Fc.T
    return P


def radio_freq(b, i):
    """The TOAs' radio frequencies [MHz] of pulsar ``i`` in engine order, read from its TOA table."""
    col = b.psrs[i].toas.table["freq"]
    return np.asarray(getattr(col, "value", col), dtype=float)[b.order[i]]


def chrom_blocks(b, i):
    """Per chromatic process of pulsar ``i``: (w ⊙ F_s [n, J] long double, phi_s [J] long double) with the weight
    restated from its definition, w = (fref / nu)^idx on the table's radio frequencies, (idx, fref) as recorded by
    ``Edge.dm`` / ``Edge.chrom`` (or set in ``b._ref_chrom[(slot, i)]`` by the caller: a process without a record is an
    error, not an assumed default); the frequencies and sqrt-priors are the recipe's fp64 parameters, as for the red
    noise."""
    out = []
    rec = getattr(b, "_ref_chrom", {})
    for slot, c in enumerate(getattr(b, "_chrom", ())):
        if c is None or c["f"][i] is None:
            continue
        if (slot, i) not in rec:
            raise ValueError(f"chromatic slot {slot} of pulsar {i} has no recorded (idx, fref): register it through "
                             "Edge.dm / Edge.chrom or record it in b._ref_chrom")
        idx, fref = rec[(slot, i)]
        w = (LD(fref) / radio_freq(b, i).astype(LD)) ** LD(idx)
        out.append((w[:, None] * basis(b.t_tdb[i], c["f"][i]).astype(LD),
                    np.asarray(c["scale"][i], dtype=float).astype(LD) ** 2))
    return out


def ld_cholesky(A):
    """Lower L with L L^T = A, long double, one column at a time."""
    n = len(A)
    L = np.zeros_like(A)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0:
            raise ValueError(f"long-double Cholesky: pivot {j} is {d}")
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _tri(L, B):
    """(L L^T)^-1 B by a forward and a backward column loop."""
    n = len(L)
    Y = np.zeros(B.shape, dtype=LD)
    for k in range(n):
        Y[k] = (B[k] - L[k, :k] @ Y[:k]) / L[k, k]
    X = np.zeros_like(Y)
    for k in reversed(range(n)):
        X[k] = (Y[k] - L[k + 1:, k] @ X[k + 1:]) / L[k, k]
    return X


def spd_solve(A, B, L=None, steps=2):
    """A^-1 B (A symmetric positive definite, long double) with ``steps`` rounds of iterative refinement."""
    L = ld_cholesky(A) if L is None else L
    X = _tri(L, B)
    for _ in range(steps):
        X = X + _tri(L, B - A @ X)
    return X


def design(b, i, tm):
    """The timing design matrix [n, k] (engine order, fp64) of ``tm`` = dict(poly, jumps, extra, dm), or None: the
    columns ``set_timing_model`` documents (1, x, .., x^poly in x = (t - t_mid) / (t_span / 2); one indicator per flag
    value, the earliest group dropped with a polynomial; ``extra`` in table order; (1400 / nu)^2 x^d, d = 0..dm)."""
    if tm is None:
        return None
    t, n = b.t_tdb[i], b.ntoa[i]
    cols = []
    half = 0.5 * (t.max() - t.min())
    x = (t - 0.5 * (t.max() + t.min())) / half
    if tm.get("poly") is not None:
        cols += [x ** d for d in range(int(tm["poly"]) + 1)]
    if tm.get("jumps") is not None:
        fl = b.psrs[i].toas.table["flags"]
        fv = [fl[j].get(tm["jumps"]) for j in b.order[i]]
        groups = list(dict.fromkeys(fv))
        for g in (groups[1:] if tm.get("poly") is not None else groups):
            cols.append(np.array([v == g for v in fv], dtype=float))
    if tm.get("extra") is not None:
        ex = np.asarray(tm["extra"], dtype=float).reshape(n, -1)
        cols += list(ex[b.order[i]].T)
    if tm.get("dm") is not None:
        w = (1400.0 / radio_freq(b, i)) ** 2
        cols += [w * x ** d for d in range(int(tm["dm"]) + 1)]
    return np.stack(cols, axis=1) if cols else None


def tier1(b, i, F, common=None, tm=None, own_red=True):
    """C_a [n, m] = P_a^-1 F with the timing model ``tm`` marginalised (constrained form), long double; in mpmath for
    pulsars of at most MP_TOAS TOAs, where a timing model that takes all but a few TOAs makes C_a a difference of
    terms up to 1e17 times larger.  ``own_red`` as for ``covariance``."""
    if b.ntoa[i] <= MP_TOAS:
        return _tier1_mp(b, i, F, common, tm, own_red)
    return dense_pinv(b, i, F, common, tm, own_red)


def dense_pinv(b, i, F, common=None, tm=None, own_red=True):
    """P_a^-1 F in long double (Cholesky of the dense ``covariance``, two steps of refinement per solve) with the timing
    model ``tm`` marginalised in the constrained form."""
    A = covariance(b, i, common, own_red)
    L = ld_cholesky(A)
    M = design(b, i, tm)
    if M is None:
        return spd_solve(A, F.astype(LD), L)
    m = F.shape[1]
    Y = spd_solve(A, np.concatenate([F, M], axis=1).astype(LD), L)
    PF, PM = Y[:, :m], Y[:, m:]
    G = M.astype(LD).T @ PM
    G = (G + G.T) / 2
    return PF - PM @ spd_solve(G, M.astype(LD).T @ PF)


MP_TOAS = 16


def _tier1_mp(b, i, F, common, tm, own_red=True):
    with mp.workdps(DPS):
        A = mp.matrix(mpmat(covariance(b, i, common, own_red)))
        Fm = mp.matrix(mpmat(F))
        M = design(b, i, tm)
        PF = _m_lu(A, Fm)
        if M is not None:
            Mm = mp.matrix(mpmat(M))
            PM = _m_lu(A, Mm)
            PF = PF - PM * _m_lu(Mm.T * PM, Mm.T * PF)
        out = np.empty(F.shape, dtype=LD)
        for r in range(F.shape[0]):
            for c in range(F.shape[1]):
                hi = float(PF[r, c])
                out[r, c] = LD(hi) + LD(float(PF[r, c] - hi))
    return out


def woodbury_cond(b, i, common=None, tm=None, own_red=True):
    """kappa_2 of the unit-diagonal S = Phi^-1 + T^T N^-1 T, T = [M, F_red, w ⊙ F_chromatic.., F_common], Phi^-1 =
    [0, 1/phi_red, 1/phi_chromatic.., 1/phi_common] (1 without any block): the conditioning of the system the
    product's Woodbury form solves.  ``own_red`` as for ``covariance``."""
    blocks, ip = [], []
    M = design(b, i, tm)
    if M is not None:
        blocks.append(M)
        ip.append(np.zeros(M.shape[1], dtype=LD))
    if own_red and b._red is not None and b._red["f"][i] is not None:
        blocks.append(basis(b.t_tdb[i], b._red["f"][i]))
        ip.append(1 / np.asarray(b._red["scale"][i], dtype=float).astype(LD) ** 2)
    for Fw, phi in chrom_blocks(b, i):
        blocks.append(Fw)
        ip.append(1 / phi)
    if common is not None:
        blocks.append(common[0])
        ip.append(1 / common[1])
    if not blocks:
        return 1.0
    T = np.concatenate(blocks, axis=1).astype(LD)
    N = noise_cov(b, i)
    S = T.T @ spd_solve(N, T, steps=0) + np.diag(np.concatenate(ip))
    sc = 1 / np.sqrt(np.diag(S))
    return float(np.linalg.cond((S * sc[:, None] * sc[None, :]).astype(np.float64)))


def cancellation_cond(e, K, Tspan, own_red=True):
    """max over pulsars of max|F^T N^-1 F| / min_j Z_a,jj (long double; GW basis k / Tspan, k = 1..K, ``Tspan`` one
    value or one per pulsar): how far the red-noise, chromatic and timing-model terms the product subtracts from
    N^-1 F (Woodbury, then the projection) cancel it.  ``own_red`` as for ``covariance``."""
    b = e.b
    out = 0.0
    for i in range(b.n_psr):
        F = basis(b.t_tdb[i], np.arange(1, K + 1) / (Tspan[i] if np.ndim(Tspan) else Tspan))
        Zn = F.astype(LD).T @ spd_solve(noise_cov(b, i), F.astype(LD), steps=0)
        Z = F.astype(LD).T @ tier1(b, i, F, None, e.tm[i], own_red)
        out = max(out, float(np.max(np.abs(Zn)) / np.min(np.abs(np.diag(Z)))))
    return out


def noise_cov(b, i):
    """N_a: white + ECORR only (long double)."""
    red, chrom = b._red, b._chrom
    b._red, b._chrom = None, ()
    try:
        return covariance(b, i)
    finally:
        b._red, b._chrom = red, chrom


# ------------------------------------------------------------------ tier 2: mpmath
def mpf(v):
    """A long double or fp64 value as an mpf, exactly."""
    hi = float(v)
    return mp.mpf(hi) + mp.mpf(float(LD(v) - LD(hi)))


def mpmat(A):
    return [[mpf(v) for v in row] for row in np.asarray(A)]


def mpvec(v):
    return [mpf(x) for x in np.asarray(v)]


def m_chol(A):
    n = len(A)
    L = [[mp.mpf(0)] * n for _ in range(n)]
    for j in range(n):
        d = A[j][j] - mp.fsum(L[j][k] * L[j][k] for k in range(j))
        if not d > 0:
            raise ValueError(f"mpmath Cholesky: pivot {j} is {mp.nstr(d, 5)}")
        L[j][j] = mp.sqrt(d)
        for r in range(j + 1, n):
            L[r][j] = (A[r][j] - mp.fsum(L[r][k] * L[j][k] for k in range(j))) / L[j][j]
    return L


def m_solve(L, v):
    n = len(L)
    y = [mp.mpf(0)] * n
    for k in range(n):
        y[k] = (v[k] - mp.fsum(L[k][j] * y[j] for j in range(k))) / L[k][k]
    x = [mp.mpf(0)] * n
    for k in reversed(range(n)):
        x[k] = (y[k] - mp.fsum(L[j][k] * x[j] for j in range(k + 1, n))) / L[k][k]
    return x


def m_logdet(L):
    return 2 * mp.fsum(mp.log(L[j][j]) for j in range(len(L)))


def m_phi(freqs, gamma, Tspan):
    """phi~ per (sin, cos) column in mpmath from the fp64 frequencies, gamma and Tspan."""
    y = mp.mpf(YEAR)
    return [(mp.mpf(float(f)) * y) ** (-mp.mpf(float(gamma))) / (12 * mp.pi ** 2 * mp.mpf(Tspan)) * y ** 3
            for f in np.repeat(np.asarray(freqs, dtype=float), 2)]


def _positions(b):
    """(RA, DEC) [rad] fp64 from RAJ [h] and DECJ [deg]: the inputs of every geometric quantity."""
    return np.array([[p.loc["RAJ"] * np.pi / 12.0, p.loc["DECJ"] * np.pi / 180.0] for p in b.psrs])


def m_orf(b, orf):
    """Gamma [P][P] in mpmath: "hd" (1.5 x ln x - x / 4 + 1/2, x = (1 - cos zeta) / 2, diagonal 1), "monopole",
    "dipole" (cos zeta) from the fp64 positions, or a matrix as given."""
    P = b.n_psr
    if not isinstance(orf, str):
        return mpmat(orf)
    pos = _positions(b)
    u = [[mp.cos(mpf(d)) * mp.cos(mpf(r)), mp.cos(mpf(d)) * mp.sin(mpf(r)), mp.sin(mpf(d))] for r, d in pos]
    G = [[mp.mpf(1)] * P for _ in range(P)]
    for a in range(P):
        for c in range(P):
            if a == c or orf == "monopole":
                continue
            cz = mp.fsum(u[a][k] * u[c][k] for k in range(3))
            if orf == "dipole":
                G[a][c] = cz
            else:
                x = (1 - cz) / 2
                G[a][c] = mp.mpf("1.5") * x * mp.log(x) - x / 4 + mp.mpf("0.5")
    return G


def m_antenna(b, sky):
    """[P][S] (F+, Fx) in mpmath from the fp64 pulsar angles (polar angle pi/2 - DEC, azimuth RA, as the product
    forms them) and sky (gwtheta, gwphi); (0, 0) where 1 + Omega . p <= FE_POLE_TOL."""
    pos = _positions(b)
    out = []
    for ra, dec in pos:
        th, ph = mpf(np.pi / 2 - dec), mpf(ra)
        p = [mp.sin(th) * mp.cos(ph), mp.sin(th) * mp.sin(ph), mp.cos(th)]
        row = []
        for gt, gp in np.asarray(sky, dtype=float):
            gt, gp = mpf(gt), mpf(gp)
            mv = [mp.sin(gp), -mp.cos(gp), 0]
            nv = [-mp.cos(gt) * mp.cos(gp), -mp.cos(gt) * mp.sin(gp), mp.sin(gt)]
            om = [-mp.sin(gt) * mp.cos(gp), -mp.sin(gt) * mp.sin(gp), -mp.cos(gt)]
            den = 1 + mp.fsum(om[k] * p[k] for k in range(3))
            if den <= FE_POLE_TOL:
                row.append((mp.mpf(0), mp.mpf(0)))
                continue
            mp_, np_ = mp.fsum(mv[k] * p[k] for k in range(3)), mp.fsum(nv[k] * p[k] for k in range(3))
            row.append(((mp_ * mp_ - np_ * np_) / (2 * den), mp_ * np_ / den))
        out.append(row)
    return out


def _f(x):
    return np.array(x, dtype=float) if not isinstance(x, mp.mpf) else float(x)


# ------------------------------------------------------------------ statistics
def _rows_of(b, rows, i):
    return rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]].astype(LD)


def _gw_tier1(e, rows, K, Tspan, common_log10_A=None, gamma=None, given=None):
    """Per pulsar (C, Z, X) of the GW basis k / Tspan, k = 1..K, long double; ``given``: per pulsar an fp64 C_a to use
    instead of tier 1's (the plan's own, to evaluate tier 2 on it)."""
    b = e.b
    f = np.arange(1, K + 1) / Tspan
    out = []
    for i in range(b.n_psr):
        F = basis(b.t_tdb[i], f)
        common = None if common_log10_A is None else (F, ld_phi(f, gamma, Tspan, common_log10_A))
        C = tier1(b, i, F, common, e.tm[i]) if given is None else np.asarray(given[i], dtype=np.float64).astype(LD)
        out.append((C, F.astype(LD).T @ C, _rows_of(b, rows, i) @ C))
    return f, out


def curn(e, rows, given=None):
    """dict(lnl [R, Ng, NA], ldet [Ng, NA], scale [R, Ng, NA] = 1 + Q/2 + ldet/2, Z [P, 2K, 2K], C) of the CURN
    registration ``e.stats["curn"]``; ``given``: evaluate tier 2 on these C_a (see ``_gw_tier1``)."""
    o, b = e.stats["curn"], e.b
    Tspan = array_tspan(b, o["Tspan"])
    f, t1 = _gw_tier1(e, rows, o["K"], Tspan, given=given)
    x, gam = o["log10_A"], o["gamma"]
    R, nc = rows.shape[0], 2 * o["K"]
    lnl, Q = np.zeros((R, len(gam), len(x))), np.zeros((R, len(gam), len(x)))
    ldet = np.zeros((len(gam), len(x)))
    with mp.workdps(DPS):
        for C, Z, X in t1:
            Zm, Xm = mpmat(Z), [mpvec(r) for r in X]
            for g, gm in enumerate(gam):
                sp = [mp.sqrt(v) for v in m_phi(f, gm, Tspan)]
                Zh = [[sp[j] * Zm[j][k] * sp[k] for k in range(nc)] for j in range(nc)]
                Xh = [[sp[j] * r[j] for j in range(nc)] for r in Xm]
                for k, xa in enumerate(x):
                    a2 = mp.mpf(10) ** (2 * mpf(xa))
                    L = m_chol([[(1 if j == c else 0) + a2 * Zh[j][c] for c in range(nc)] for j in range(nc)])
                    ld = m_logdet(L)
                    ldet[g, k] += float(ld)
                    for r in range(R):
                        q = a2 * mp.fsum(u * v for u, v in zip(Xh[r], m_solve(L, Xh[r])))
                        lnl[r, g, k] += float(q / 2 - ld / 2)
                        Q[r, g, k] += float(q)
    return dict(lnl=lnl, ldet=ldet, scale=1 + 0.5 * Q + 0.5 * ldet[None], C=[c for c, _, _ in t1],
                Z=np.stack([z for _, z, _ in t1]).astype(np.float64))


def hd(e, rows, given=None):
    """dict(lnl, ldet, scale) of the HD registration ``e.stats["hd"]`` on the CURN grid: the stacked system of
    N = P 2K, ln L = 1/2 y^T (I + M)^-1 y - 1/2 ln det(I + M), M = G^T Z G, y = G^T X, G = A (B (x) phi~^1/2), B B^T =
    Gamma from an mpmath eigendecomposition (eigenvalues below zero, rounding of an fp64 PSD matrix, set to 0);
    ``given`` as for ``curn``."""
    o, b = e.stats["curn"], e.b
    Tspan = array_tspan(b, o["Tspan"])
    f, t1 = _gw_tier1(e, rows, o["K"], Tspan, given=given)
    x, gam = o["log10_A"], o["gamma"]
    P, R, nc = b.n_psr, rows.shape[0], 2 * o["K"]
    N = P * nc
    lnl, Q = np.zeros((R, len(gam), len(x))), np.zeros((R, len(gam), len(x)))
    ldet = np.zeros((len(gam), len(x)))
    with mp.workdps(DPS):
        mu, E = mp.eigsy(mp.matrix(m_orf(b, e.stats["hd"])))
        B = [[E[a, j] * mp.sqrt(max(mu[j], 0)) for j in range(P)] for a in range(P)]
        BB = [[[B[a][j] * B[a][c] for c in range(P)] for j in range(P)] for a in range(P)]
        Zm = [mpmat(z) for _, z, _ in t1]
        Xm = [[mpvec(r) for r in X] for _, _, X in t1]
        for g, gm in enumerate(gam):
            sp = [mp.sqrt(v) for v in m_phi(f, gm, Tspan)]
            Zh = [[[sp[j] * Z[j][k] * sp[k] for k in range(nc)] for j in range(nc)] for Z in Zm]
            M0 = [[mp.fsum(BB[a][j // nc][c // nc] * Zh[a][j % nc][c % nc] for a in range(P)) for c in range(N)]
                  for j in range(N)]
            y0 = [[mp.fsum(B[a][j // nc] * sp[j % nc] * Xm[a][r][j % nc] for a in range(P)) for j in range(N)]
                  for r in range(R)]
            for k, xa in enumerate(x):
                a2 = mp.mpf(10) ** (2 * mpf(xa))
                L = m_chol([[(1 if j == c else 0) + a2 * M0[j][c] for c in range(N)] for j in range(N)])
                ld = m_logdet(L)
                ldet[g, k] = float(ld)
                for r in range(R):
                    q = a2 * mp.fsum(u * v for u, v in zip(y0[r], m_solve(L, y0[r])))
                    lnl[r, g, k] = float(q / 2 - ld / 2)
                    Q[r, g, k] = float(q)
    return dict(lnl=lnl, ldet=ldet, scale=1 + 0.5 * Q + 0.5 * ldet[None])


def _os_pairs(e, rows):
    """The optimal statistic's tier 2 common part: (pairs, t [n_pairs], d [R, n_pairs], |x_a||x_b| [R, n_pairs]) in
    mpmath, plus the long-double C and Z per pulsar."""
    o, b = e.stats["os"], e.b
    Tspan = array_tspan(b, o["Tspan"])
    f, t1 = _gw_tier1(e, rows, o["K"], Tspan, o["log10_A_common"], o["gamma"])
    P, R, nc = b.n_psr, rows.shape[0], 2 * o["K"]
    pa, pb = np.triu_indices(P, 1)
    phi = m_phi(f, o["gamma"], Tspan)
    Zh = [[[phi[j] * v for v in row] for j, row in enumerate(mpmat(z))] for _, z, _ in t1]    # phi~ Z
    x = [[[mp.sqrt(phi[j]) * v for j, v in enumerate(mpvec(r))] for r in X] for _, _, X in t1]
    t = [mp.fsum(Zh[a][j][k] * Zh[c][k][j] for j in range(nc) for k in range(nc)) for a, c in zip(pa, pb)]
    d = [[mp.fsum(u * v for u, v in zip(x[a][r], x[c][r])) for a, c in zip(pa, pb)] for r in range(R)]
    nx = [[mp.sqrt(mp.fsum(v * v for v in x[a][r])) for a in range(P)] for r in range(R)]
    dn = [[nx[r][a] * nx[r][c] for a, c in zip(pa, pb)] for r in range(R)]
    return (pa, pb), t, d, dn, t1


def optimal_statistic(e, rows):
    """dict(rho, A2, snr, A2_mc (each [R, ...]) and their scales, t_ab, finv, C, Z) of ``e.stats["os"]``."""
    o, b = e.stats["os"], e.b
    with mp.workdps(DPS):
        (pa, pb), t, d, dn, t1 = _os_pairs(e, rows)
        W = [[Gm[a][c] for a, c in zip(pa, pb)] for Gm in (m_orf(b, g) for g in o["orfs"])]
        no, nq, R = len(W), len(t), rows.shape[0]
        D = [mp.fsum(w[q] ** 2 * t[q] for q in range(nq)) for w in W]
        Fm = mp.matrix([[mp.fsum(W[i][q] * W[j][q] * t[q] for q in range(nq)) for j in range(no)] for i in range(no)])
        Fi = Fm ** -1
        out = dict(rho=[], A2=[], snr=[], A2_mc=[], rho_s=[], A2_s=[], snr_s=[], A2_mc_s=[])
        for r in range(R):
            bo = [mp.fsum(W[i][q] * d[r][q] for q in range(nq)) for i in range(no)]
            bs = [mp.fsum(abs(W[i][q]) * dn[r][q] for q in range(nq)) for i in range(no)]
            out["rho"].append([d[r][q] / t[q] for q in range(nq)])
            out["rho_s"].append([dn[r][q] / t[q] for q in range(nq)])
            out["A2"].append([bo[i] / D[i] for i in range(no)])
            out["A2_s"].append([bs[i] / D[i] for i in range(no)])
            out["snr"].append([bo[i] / mp.sqrt(D[i]) for i in range(no)])
            out["snr_s"].append([bs[i] / mp.sqrt(D[i]) for i in range(no)])
            out["A2_mc"].append([mp.fsum(Fi[i, j] * bo[j] for j in range(no)) for i in range(no)])
            out["A2_mc_s"].append([mp.fsum(abs(Fi[i, j]) * bs[j] for j in range(no)) for i in range(no)])
        out = {k: np.array([[float(v) for v in row] for row in val]) for k, val in out.items()}
        out.update(t_ab=np.array([float(v) for v in t]), finv=np.array([[float(Fi[i, j]) for j in range(no)] for i in range(no)]),
                   C=[c for c, _, _ in t1], Z=np.stack([z for _, z, _ in t1]).astype(np.float64))
    return out


def pfos(e, rows):
    """dict(rho [R, K, n_pairs], phi, snr, phi_mc [R, n_orf, K], their scales, t [K, n_pairs], D [n_orf, K]) of the
    per-frequency optimal statistic on ``e.stats["os"]``, in the units of the unscaled projection: Z_a[k] the 2 x 2
    diagonal block of Z_a at f_k, X_a,k the projection pair, t_qk = tr(Z_a[k] Z_b[k]), d_qk = X_a,k . X_b,k,
    D_ok = sum_q (Gamma^o_q)^2 t_qk, (F_k)_oo' = sum_q Gamma^o_q Gamma^o'_q t_qk; scales |X_a,k||X_b,k| and their
    template sums, as ``optimal_statistic``."""
    o, b = e.stats["os"], e.b
    Tspan = array_tspan(b, o["Tspan"])
    _, t1 = _gw_tier1(e, rows, o["K"], Tspan, o["log10_A_common"], o["gamma"])
    K, P, R = o["K"], b.n_psr, rows.shape[0]
    pa, pb = np.triu_indices(P, 1)
    nq, no = len(pa), len(o["orfs"])
    out = {k: np.zeros((R, K, nq)) for k in ("rho", "rho_s")}
    out.update({k: np.zeros((R, no, K)) for k in ("phi", "phi_s", "snr", "snr_s", "phi_mc", "phi_mc_s")})
    tt, DD = np.zeros((K, nq)), np.zeros((no, K))
    with mp.workdps(DPS):
        W = [[Gm[a][c] for a, c in zip(pa, pb)] for Gm in (m_orf(b, g) for g in o["orfs"])]
        Zm = [mpmat(z) for _, z, _ in t1]
        Xm = [[mpvec(r) for r in X] for _, _, X in t1]
        for k in range(K):
            c2 = (2 * k, 2 * k + 1)
            t = [mp.fsum(Zm[a][u][v] * Zm[c][v][u] for u in c2 for v in c2) for a, c in zip(pa, pb)]
            D = [mp.fsum(w[q] ** 2 * t[q] for q in range(nq)) for w in W]
            Fi = mp.matrix([[mp.fsum(W[i][q] * W[j][q] * t[q] for q in range(nq)) for j in range(no)]
                            for i in range(no)]) ** -1
            tt[k], DD[:, k] = [float(v) for v in t], [float(v) for v in D]
            for r in range(R):
                d = [mp.fsum(Xm[a][r][u] * Xm[c][r][u] for u in c2) for a, c in zip(pa, pb)]
                nx = [mp.sqrt(mp.fsum(Xm[a][r][u] ** 2 for u in c2)) for a in range(P)]
                dn = [nx[a] * nx[c] for a, c in zip(pa, pb)]
                bo = [mp.fsum(W[i][q] * d[q] for q in range(nq)) for i in range(no)]
                bs = [mp.fsum(abs(W[i][q]) * dn[q] for q in range(nq)) for i in range(no)]
                out["rho"][r, k] = [float(d[q] / t[q]) for q in range(nq)]
                out["rho_s"][r, k] = [float(dn[q] / t[q]) for q in range(nq)]
                for i in range(no):
                    out["phi"][r, i, k], out["phi_s"][r, i, k] = float(bo[i] / D[i]), float(bs[i] / D[i])
                    out["snr"][r, i, k], out["snr_s"][r, i, k] = float(bo[i] / mp.sqrt(D[i])), float(bs[i] / mp.sqrt(D[i]))
                    out["phi_mc"][r, i, k] = float(mp.fsum(Fi[i, j] * bo[j] for j in range(no)))
                    out["phi_mc_s"][r, i, k] = float(mp.fsum(abs(Fi[i, j]) * bs[j] for j in range(no)))
    out.update(t=tt, D=DD)
    return out


def rn_spans(e):
    """T_a per pulsar of ``e.stats["rn"]``: its Tspan, else the pulsar's own span."""
    o, b = e.stats["rn"], e.b
    return [float(o["Tspan"]) if o["Tspan"] is not None else float(t.max() - t.min()) for t in b.t_tdb]


def rn(e, rows, given=None):
    """dict(lnl [R, P, Ng, NA], ldet [P, Ng, NA], scale = 1 + Q/2 + ldet/2, C, Z [P, 2K, 2K]) of the red-noise
    likelihood ``e.stats["rn"]``: per pulsar the basis F_a at k / T_a, C_a = P_a^-1 F_a with the pulsar's own red noise
    out of P_a (its chromatic processes and the optional common power law at k / Tspan of the array in it), Z_a =
    F_a^T C_a, X_a = C_a^T r, and per grid point ln L_a = 1/2 y^T (I + M)^-1 y - 1/2 ln det(I + M), M = A^2 phi~^1/2
    Z_a phi~^1/2, y = A phi~^1/2 X_a (phi~ the set_red power law at T_a); ``given`` as for ``curn``."""
    o, b = e.stats["rn"], e.b
    x, gam = o["log10_A"], o["gamma"]
    P, R, nc = b.n_psr, rows.shape[0], 2 * o["K"]
    TA = array_tspan(b)
    fc = np.arange(1, o["components_common"] + 1) / TA
    lnl, Q = np.zeros((R, P, len(gam), len(x))), np.zeros((R, P, len(gam), len(x)))
    ldet = np.zeros((P, len(gam), len(x)))
    Cs, Zs = [], []
    with mp.workdps(DPS):
        for i, Ta in enumerate(rn_spans(e)):
            f = np.arange(1, o["K"] + 1) / Ta
            F = basis(b.t_tdb[i], f)
            common = None if o["log10_A_common"] is None else \
                (basis(b.t_tdb[i], fc), ld_phi(fc, o["gamma_common"], TA, o["log10_A_common"]))
            C = tier1(b, i, F, common, e.tm[i], own_red=False) if given is None else \
                np.asarray(given[i], dtype=np.float64).astype(LD)
            Z, X = F.astype(LD).T @ C, _rows_of(b, rows, i) @ C
            Cs.append(C)
            Zs.append(Z)
            Zm, Xm = mpmat(Z), [mpvec(r) for r in X]
            for g, gm in enumerate(gam):
                sp = [mp.sqrt(v) for v in m_phi(f, gm, Ta)]
                Zh = [[sp[j] * Zm[j][k] * sp[k] for k in range(nc)] for j in range(nc)]
                Xh = [[sp[j] * r[j] for j in range(nc)] for r in Xm]
                for k, xa in enumerate(x):
                    a2 = mp.mpf(10) ** (2 * mpf(xa))
                    L = m_chol([[(1 if j == c else 0) + a2 * Zh[j][c] for c in range(nc)] for j in range(nc)])
                    ld = m_logdet(L)
                    ldet[i, g, k] = float(ld)
                    for r in range(R):
                        q = a2 * mp.fsum(u * v for u, v in zip(Xh[r], m_solve(L, Xh[r])))
                        lnl[r, i, g, k] = float(q / 2 - ld / 2)
                        Q[r, i, g, k] = float(q)
    return dict(lnl=lnl, ldet=ldet, scale=1 + 0.5 * Q + 0.5 * ldet[None], C=Cs, Z=np.stack(Zs).astype(np.float64))


def anisotropy(e, rows, templates_sph=None):
    """dict(clm [R, n_lm], chi2 [R], radio [R, S] and their scales) of ``e.stats["aniso"]`` (lmax, sky) on the optimal
    statistic: F = T diag(t) T^T, c = F^-1 T d, chi2 = y^T F^-1 y - y_0^2 / F_00 (y = T d), S/N_k = y_k / sqrt(F_kk).
    ``templates_sph``: [n_lm, n_pairs] fp64 spherical-harmonic templates (the set_gwb basis; their definition is pinned
    to the reference project elsewhere); the radiometer's come from ``m_antenna``."""
    o, b = e.stats["aniso"], e.b
    out = {}
    with mp.workdps(DPS):
        (pa, pb), t, d, dn, _ = _os_pairs(e, rows)
        nq, R = len(t), rows.shape[0]
        if templates_sph is not None:
            T = mpmat(templates_sph)
            n = len(T)
            F = mp.matrix([[mp.fsum(T[i][q] * T[j][q] * t[q] for q in range(nq)) for j in range(n)] for i in range(n)])
            Fi = F ** -1
            clm, chi2, cs = [], [], []
            for r in range(R):
                y = [mp.fsum(T[i][q] * d[r][q] for q in range(nq)) for i in range(n)]
                ys = [mp.fsum(abs(T[i][q]) * dn[r][q] for q in range(nq)) for i in range(n)]
                c = [mp.fsum(Fi[i, j] * y[j] for j in range(n)) for i in range(n)]
                clm.append([float(v) for v in c])
                cs.append([float(mp.fsum(abs(Fi[i, j]) * ys[j] for j in range(n))) for i in range(n)])
                full = mp.fsum(y[i] * c[i] for i in range(n))
                chi2.append((float(full - y[0] ** 2 / F[0, 0]), float(full)))
            out.update(clm=np.array(clm), clm_s=np.array(cs), chi2=np.array(chi2)[:, 0], chi2_s=np.array(chi2)[:, 1])
        if o.get("sky") is not None:
            ant = m_antenna(b, o["sky"])
            S = len(o["sky"])
            Tr = [[mp.mpf("1.5") / S * (ant[a][k][0] * ant[c][k][0] + ant[a][k][1] * ant[c][k][1])
                   for a, c in zip(pa, pb)] for k in range(S)]
            Fkk = [mp.fsum(Tr[k][q] ** 2 * t[q] for q in range(nq)) for k in range(S)]
            out["radio"] = np.array([[float(mp.fsum(Tr[k][q] * d[r][q] for q in range(nq)) / mp.sqrt(Fkk[k]))
                                      for k in range(S)] for r in range(R)])
            out["radio_s"] = np.array([[float(mp.fsum(abs(Tr[k][q]) * dn[r][q] for q in range(nq)) / mp.sqrt(Fkk[k]))
                                        for k in range(S)] for r in range(R)])
    return out


def fp(e, rows):
    """dict(Fp [R, Nf], amps [R, P, Nf, 2] (X^ = L^-1 N, L the lower Cholesky factor of M_a(f)), N [R, P, Nf, 2]
    (C_a(f)^T r), M [P, Nf, 2, 2] (long double, as fp64), lmin_info [P, Nf] (lambda_min(M) / sum 1/sigma^2), kappa
    [P, Nf] of M_a(f)) of ``e.stats["fp"]``."""
    o, b = e.stats["fp"], e.b
    f = o["freqs"]
    Nf, P, R = len(f), b.n_psr, rows.shape[0]
    Tspan = array_tspan(b, o["Tspan"])
    fc = np.arange(1, o["components_common"] + 1) / Tspan
    amps, Ns = np.zeros((R, P, Nf, 2)), np.zeros((R, P, Nf, 2))
    Ms, lmin, kap = np.zeros((P, Nf, 2, 2)), np.zeros((P, Nf)), np.zeros((P, Nf))
    Mm, Nm = [], []
    with mp.workdps(DPS):
        for i in range(P):
            t = b.t_tdb[i]
            F = basis(t, f)
            common = None if o["log10_A_common"] is None else \
                (basis(t, fc), ld_phi(fc, o["gamma_common"], Tspan, o["log10_A_common"]))
            C = tier1(b, i, F, common, e.tm[i])
            Nr = _rows_of(b, rows, i) @ C
            w1, w2 = (np.asarray(v, dtype=float) for v in b._white[i])
            info = mp.fsum(1 / mpf(v) for v in (w1 * w1 + w2 * w2))
            Mi, Ni = [], []
            for k in range(Nf):
                c = slice(2 * k, 2 * k + 2)
                M = F[:, c].astype(LD).T @ C[:, c]
                M = mpmat((M + M.T) / 2)
                Ms[i, k] = np.array([[float(v) for v in row] for row in M])
                ev = mp.eigsy(mp.matrix(M))[0]
                lmin[i, k], kap[i, k] = float(ev[0] / info), float(ev[1] / ev[0])
                L = m_chol(M)
                Mi.append(M)
                Ni.append([mpvec(Nr[r, c]) for r in range(R)])
                for r in range(R):
                    n_ = Ni[-1][r]
                    Ns[r, i, k] = [float(v) for v in n_]
                    x0 = n_[0] / L[0][0]
                    amps[r, i, k] = float(x0), float((n_[1] - L[1][0] * x0) / L[1][1])
            Mm.append(Mi)
            Nm.append(Ni)
        Fp = 0.5 * np.sum(amps ** 2, axis=(1, 3))
    return dict(Fp=Fp, amps=amps, N=Ns, M=Ms, lmin_info=lmin, kappa=kap, _M=Mm, _N=Nm)


def fe(e, rows, rf=None):
    """dict(Fe [R, Nf, S], kappa [Nf, S] of M4) of ``e.stats["fe"]`` (sky) on the Fp registration: M4 = sum_a e_a e_a^T
    (x) M_a(f), N4 = sum_a e_a (x) N_a(f), Fe = 1/2 N4^T M4^-1 N4 (index 2 pol + c)."""
    b = e.b
    rf = fp(e, rows) if rf is None else rf
    sky = e.stats["fe"]["sky"]
    P, R, Nf, S = b.n_psr, rows.shape[0], rf["Fp"].shape[1], len(sky)
    out, kap = np.zeros((R, Nf, S)), np.zeros((Nf, S))
    with mp.workdps(DPS):
        ant = m_antenna(b, sky)
        for k in range(Nf):
            for s in range(S):
                M4 = [[mp.fsum(ant[a][s][p // 2] * ant[a][s][q // 2] * rf["_M"][a][k][p % 2][q % 2] for a in range(P))
                       for q in range(4)] for p in range(4)]
                ev = mp.eigsy(mp.matrix(M4))[0]
                kap[k, s] = float(ev[3] / ev[0])
                L = m_chol(M4)
                for r in range(R):
                    n4 = [mp.fsum(ant[a][s][p // 2] * rf["_N"][a][k][r][p % 2] for a in range(P)) for p in range(4)]
                    out[r, k, s] = float(mp.fsum(u * v for u, v in zip(n4, m_solve(L, n4))) / 2)
    return dict(Fe=out, kappa=kap, Fp=rf["Fp"])


def self_check(e):
    """Tier 1 of pulsar 0 of ``e`` (CURN's basis) entirely in mpmath (dense P_a, mpmath LU solves, the constrained
    timing-model form): the long-double C's worst |d| / max|C|."""
    b, o = e.b, e.stats["curn"]
    Tspan = array_tspan(b, o["Tspan"])
    F = basis(b.t_tdb[0], np.arange(1, o["K"] + 1) / Tspan)
    global MP_TOAS
    keep, MP_TOAS = MP_TOAS, 0
    try:
        C = tier1(b, 0, F, None, e.tm[0])
    finally:
        MP_TOAS = keep
    with mp.workdps(DPS):
        A = mp.matrix(mpmat(covariance(b, 0)))
        Fm = mp.matrix(mpmat(F))
        M = design(b, 0, e.tm[0])
        PF = _m_lu(A, Fm)
        if M is not None:
            Mm = mp.matrix(mpmat(M))
            PM = _m_lu(A, Mm)
            PF = PF - PM * _m_lu(Mm.T * PM, Mm.T * PF)
        ref = np.array([[float(PF[r, c]) for c in range(F.shape[1])] for r in range(F.shape[0])])
        diff = np.array([[float(mpf(C[r, c]) - PF[r, c]) for c in range(F.shape[1])] for r in range(F.shape[0])])
    return float(np.max(np.abs(diff)) / np.max(np.abs(ref)))


def _m_lu(A, B):
    """A^-1 B for an mpmath matrix B, one column at a time."""
    X = mp.matrix(A.rows, B.cols)
    for c in range(B.cols):
        x = mp.lu_solve(A, B.column(c))
        for r in range(A.rows):
            X[r, c] = x[r]
    return X


# ------------------------------------------------------------------ edge recipes
PLAN_ONLY = True          # recipes build plan_only batches; the device tests set False


class Edge:
    """A ``plan_only`` PulsarBatch with its name, each pulsar's timing-model columns ``tm`` (None or dict(poly,
    jumps, extra)) and the statistics' settings ``stats`` -- what the reference reads besides the batch's noise
    recipe (_white, _ecorr, _red, TOA times, flags and positions)."""

    def __init__(self, name, psrs):
        from pta_replicator_b200.engine import PulsarBatch
        self.name = name
        self.b = PulsarBatch(psrs, plan_only=PLAN_ONLY)
        self.b._ref_chrom = {}
        self.tm = [None] * self.b.n_psr
        self.stats = {}

    def timing_model(self, i, poly=2, jumps=None, extra=None, dm=None):
        self.b.set_timing_model(i, poly=poly, jumps=jumps, extra=extra, dm=dm)
        self.tm[i] = dict(poly=poly, jumps=jumps, extra=extra, dm=dm)

    def dm(self, i, log10_A, gamma, components, modes=None, fref=1400.0):
        """DM noise on pulsar ``i``; the reference restates its weight from (idx = 2, ``fref``)."""
        self.b.set_dm_noise(i, log10_A, gamma, components=components, modes=modes, fref=fref)
        self.b._ref_chrom[(0, i)] = (2.0, fref)
        return self

    def chrom(self, i, log10_A, gamma, components, idx=4.0, modes=None, fref=1400.0):
        """A chromatic (scattering, idx 4) process on pulsar ``i``; the reference restates its weight from (idx, fref)."""
        self.b.set_chromatic_noise(i, log10_A, gamma, idx=idx, components=components, modes=modes, fref=fref)
        self.b._ref_chrom[(1, i)] = (float(idx), fref)
        return self

    def rn(self, K, log10_A=(-15.0, -12.5, -11.0), gamma=(1.0, 4.0, 6.5), Tspan=None, log10_A_common=None,
           gamma_common=13 / 3, components_common=14):
        """The red-noise likelihood on a 3 x 3 grid, optionally with a common power law in P_a."""
        x, g = np.array(log10_A, dtype=float), np.array(gamma, dtype=float)
        self.b.set_red_noise_likelihood(log10_A=x, gamma=g, components=K, Tspan=Tspan, log10_A_common=log10_A_common,
                                        gamma_common=gamma_common, components_common=components_common)
        self.stats["rn"] = dict(K=K, log10_A=x, gamma=g, Tspan=Tspan, log10_A_common=log10_A_common,
                                gamma_common=gamma_common, components_common=components_common)
        return self

    def pfos(self):
        """The per-frequency optimal statistic on the ``os`` registration."""
        self.b.set_os_per_frequency()
        self.stats["os"]["pf"] = True
        return self

    def curn(self, K, log10_A=(-18.0, -12.0, -11.0), gamma=(0.0, 7.0), Tspan=None, hd=None):
        x, g = np.array(log10_A, dtype=float), np.array(gamma, dtype=float)
        self.b.set_curn_likelihood(log10_A=x, gamma=g, components=K, Tspan=Tspan)
        self.stats["curn"] = dict(K=K, log10_A=x, gamma=g, Tspan=Tspan)
        if hd is not None:
            self.b.set_hd_likelihood(hd)
            self.stats["hd"] = hd
        return self

    def os(self, K, orfs=("hd", "monopole", "dipole"), gamma=13 / 3, log10_A_common=None, Tspan=None, lmax=None,
           sky=None):
        self.b.set_optimal_statistic(components=K, gamma=gamma, orfs=orfs, log10_A_common=log10_A_common, Tspan=Tspan)
        self.stats["os"] = dict(K=K, orfs=orfs, gamma=gamma, log10_A_common=log10_A_common, Tspan=Tspan)
        if lmax is not None or sky is not None:
            self.b.set_os_anisotropy(lmax=lmax, sky=sky)
            self.stats["aniso"] = dict(lmax=lmax, sky=sky)
        return self

    def fp(self, freqs=None, n_freqs=4, Tspan=None, log10_A_common=None, gamma_common=13 / 3, components_common=14,
           sky=None):
        f = np.arange(1, n_freqs + 1) / array_tspan(self.b, Tspan) if freqs is None else np.asarray(freqs, dtype=float)
        self.b.set_fp_statistic(freqs=f, Tspan=Tspan, log10_A_common=log10_A_common, gamma_common=gamma_common,
                                components_common=components_common)
        self.stats["fp"] = dict(freqs=f, Tspan=Tspan, log10_A_common=log10_A_common, gamma_common=gamma_common,
                                components_common=components_common)
        if sky is not None:
            self.b.set_fe_statistic(sky=sky)
            self.stats["fe"] = dict(sky=np.asarray(sky, dtype=float))
        return self


def pulsars(ntoas, seed=0, err_us=None, pos=None, jump_single=False, name="T", radio=False, single=(), spans={}):
    """Synthetic pulsars with the given TOA counts: epochs of 1-4 TOAs within 1 s over MJD 53000-58800, backends A/B/C
    cycling per epoch (flag f), uncertainties 0.3-3 us (or ``err_us(rng, n)``), isotropic positions (or ``pos``:
    (RAJ [h], DECJ [deg]) per pulsar).  ``jump_single``: flag j = "x" on every TOA but one (index n // 2, "y").
    ``radio``: sub-band radio frequencies, each epoch's TOAs spread evenly over 700-1900 MHz (1400 MHz alone), the
    pulsars in ``single`` at 820 MHz only; they draw nothing, so the TOAs are those of ``radio`` False.  ``spans``:
    pulsar -> (first, last) MJD range of its epochs instead of 53000-58800."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, n in enumerate(ntoas):
        sub = []
        while sum(sub) < n:
            sub.append(int(min(rng.integers(1, 5), n - sum(sub))))
        ep = np.sort(rng.uniform(*spans.get(j, (53000.0, 58800.0)), len(sub)))
        mjd = np.concatenate([e + np.sort(rng.uniform(0, 0.9, k)) / 86400.0 for e, k in zip(ep, sub)])
        be = np.concatenate([[("A", "B", "C")[q % 3]] * k for q, k in enumerate(sub)])
        ra, dec = (rng.uniform(0, 24), math.degrees(math.asin(rng.uniform(-1, 1)))) if pos is None else pos[j]
        err = rng.uniform(0.3, 3.0, n) if err_us is None else err_us(rng, n)
        fl = [{"f": f, "j": "y" if (jump_single and q == n // 2) else "x"} for q, f in enumerate(be)]
        kw = {}
        if radio:
            nu = np.concatenate([np.linspace(700.0, 1900.0, k) if k > 1 else [1400.0] for k in sub])
            kw["freq"] = np.full(n, 820.0) if j in single else nu
        p = pulsar_from_arrays(f"{name}{j:03d}", {"RAJ": float(ra), "DECJ": float(dec)}, mjd.astype(np.longdouble), err,
                               flags=fl, **kw)
        make_ideal(p)
        out.append(p)
    return out


def _noise(e, white=True, ecorr=-6.3, coarsegrain=1.0 / 86400.0, red=None, tm=False):
    """White (efac 1.1, equad 10^-6.5 s), optional ECORR and red noise (log10_A, gamma, components[, modes]) and a
    timing model (``tm``: True = poly 2 + jumps on f where it fits, else a dict for set_timing_model)."""
    b = e.b
    for i in range(b.n_psr):
        if white:
            b.set_white(i, efac=1.1, log10_equad=-6.5)
        if ecorr is not None:
            b.set_ecorr(i, ecorr, coarsegrain=coarsegrain)
        if red is not None:
            b.set_red(i, red[0], red[1], components=red[2], modes=red[3] if len(red) > 3 else None)
        if tm is True and b.ntoa[i] >= 20:
            e.timing_model(i, **_largest_model(b, i))
        elif isinstance(tm, dict):
            e.timing_model(i, **tm)
    return e


def _largest_model(b, i):
    """The largest of poly 2 + jumps on f, poly 1 + jumps, offset + jumps, poly 1, offset that leaves at least three
    TOAs free (so every Fp frequency keeps two) and whose whitened columns are well conditioned (kappa < 1e6)."""
    for poly, jumps in ((2, "f"), (1, "f"), (0, "f"), (1, None), (0, None)):
        M = design(b, i, dict(poly=poly, jumps=jumps))
        if M.shape[1] <= b.ntoa[i] - 3:
            A = M / np.linalg.norm(M, axis=0)
            if np.linalg.cond(A) < 1e6:
                return dict(poly=poly, jumps=jumps)
    return dict(poly=None, jumps=None)


EDGE4 = (5, 7, 65, 193)


def rows_of(b, R=3, seed=0):
    """Engine-order rows [R, ld], zero in the alignment slots: r % 3 == 0 white draws at the TOA uncertainties, 1 the
    draws plus a 1-us sinusoid at 2 / span, 2 a 10-us sinusoid at 1 / span (a loud red signal) plus the draws."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((R, b.ld))
    span = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    for i in range(b.n_psr):
        s, n, t = b.toa_off[i], b.ntoa[i], b.t_tdb[i]
        for r in range(R):
            v = rng.standard_normal(n) * b.err_s[i]
            if r % 3 == 1:
                v = v + 1e-6 * np.sin(4 * np.pi * t / span + 0.3 * i)
            elif r % 3 == 2:
                v = v + 1e-5 * np.sin(2 * np.pi * t / span + 0.7 * i)
            rows[r, s:s + n] = v
    return rows


def near_pole_sky(b, i, rad):
    """Sky points (gwtheta, gwphi) ``rad`` from pulsar ``i``'s line of sight, offset in gwtheta and in gwphi."""
    ra, dec = _positions(b)[i]
    th = np.pi / 2 - dec
    return np.array([[th + rad, ra], [th, ra + rad / max(np.sin(th), 1e-3)]])


def recipes():
    """name -> builder() of every edge recipe; each builder returns an Edge with its registrations."""
    R = {}
    # 1. the default grid's corners, white + ECORR
    R["corners_k1"] = lambda: _noise(Edge("corners_k1", pulsars(EDGE4, 11))).curn(1, hd="hd")
    R["corners_k16"] = lambda: _noise(Edge("corners_k16", pulsars(EDGE4, 12))).curn(16)
    R["corners_k16_hd"] = lambda: _noise(Edge("corners_k16_hd", pulsars((65, 193), 13))).curn(16, hd="hd")
    # 2. rank-deficient Z_a: fewer TOAs than basis columns, with and without a model that takes most of them
    R["rankdef"] = lambda: _noise(Edge("rankdef", pulsars((5, 6, 7), 21))).curn(16).os(16, orfs=("hd",)).fp(n_freqs=3)
    def rankdef_tm():
        e = _noise(Edge("rankdef_tm", pulsars((5, 6, 7), 22)))
        for i in range(e.b.n_psr):
            e.timing_model(i, poly=0, jumps="f")
        return e.curn(16).os(16, orfs=("hd",))
    R["rankdef_tm"] = rankdef_tm
    def rankdef_hd():
        e = _noise(Edge("rankdef_hd", pulsars((5, 7), 23)))
        for i in range(e.b.n_psr):
            e.timing_model(i, poly=0, jumps="f")
        return e.curn(16, hd="hd")
    R["rankdef_hd"] = rankdef_hd
    # 3. ECORR: single-TOA buckets, one bucket per pulsar, ECORR 100-1000 sigma, per-backend with one backend at zero
    R["ecorr_single"] = lambda: _noise(Edge("ecorr_single", pulsars(EDGE4, 31)), coarsegrain=1e-12).curn(16).os(8, orfs=("hd",)).fp()
    R["ecorr_whole"] = lambda: _noise(Edge("ecorr_whole", pulsars(EDGE4, 32)), coarsegrain=1e5).curn(16).os(8, orfs=("hd",)).fp()
    R["ecorr_loud"] = lambda: _noise(Edge("ecorr_loud", pulsars(EDGE4, 33)), ecorr=-3.5, tm=True).curn(16).os(8, orfs=("hd",)).fp()

    def per_backend():
        e = _noise(Edge("ecorr_backend", pulsars(EDGE4, 34)), ecorr=None, tm=True)
        for i in range(e.b.n_psr):
            e.b.set_ecorr(i, [-6.0, -5.0, -np.inf], flags=["A", "B", "C"], coarsegrain=1.0 / 86400.0)
        return e.curn(16).os(8, orfs=("hd",)).fp()
    R["ecorr_backend"] = per_backend
    # 4. loud steep red noise, also on exactly the GW basis frequencies
    R["red_loud"] = lambda: _noise(Edge("red_loud", pulsars(EDGE4, 41)), red=(-11.5, 6.5, 30), tm=True).curn(16).os(16, orfs=("hd",)).fp()

    def red_gw_modes():
        e = Edge("red_gw_modes", pulsars(EDGE4, 42))
        T = array_tspan(e.b)
        return _noise(e, red=(-11.5, 6.5, 16, np.arange(1, 17) / T)).curn(16).os(16, orfs=("hd",)).fp()
    R["red_gw_modes"] = red_gw_modes
    R["red_loud_hd"] = lambda: _noise(Edge("red_loud_hd", pulsars(EDGE4, 43)), red=(-11.5, 6.5, 30), tm=True).curn(1, hd="dipole")

    # 5. timing model: a one-TOA jump group; an extra column nearly collinear with the 1 / Tspan sine
    def single_jump():
        e = _noise(Edge("tm_single_jump", pulsars(EDGE4, 51, jump_single=True)))
        for i in range(e.b.n_psr):
            if e.b.ntoa[i] >= 20:
                e.timing_model(i, poly=2, jumps="j")
        return e.curn(16).os(8, orfs=("hd",)).fp()
    R["tm_single_jump"] = single_jump
    R["tm_collinear"] = lambda: collinear(accept=True)

    # 6. white noise from 1e-8 s to 1e-5 s, equad added (tnequad)
    def white_span():
        e = Edge("white_span", pulsars(EDGE4, 61, err_us=lambda rng, n: 10.0 ** rng.uniform(-2, 1, n)))
        for i in range(e.b.n_psr):
            e.b.set_white(i, efac=1.0, log10_equad=-8.0, tnequad=True)
            e.b.set_ecorr(i, -7.0, coarsegrain=1.0 / 86400.0)
            if e.b.ntoa[i] >= 20:
                e.timing_model(i, **_largest_model(e.b, i))
        return e.curn(16).os(16, orfs=("hd",)).fp()
    R["white_span"] = white_span
    # 7. a loud common process in P for OS, Fp and Fe
    R["common_loud"] = lambda: _noise(Edge("common_loud", pulsars(EDGE4, 71)), tm=True).os(
        8, log10_A_common=-13.5).fp(log10_A_common=-13.5, sky=[[0.3, 1.0], [1.7, 4.0], [2.9, 5.5]])

    # 8. Tspan overrides, 0.5 and 2 times the data span
    def tspan(fac):
        e = _noise(Edge(f"tspan_{fac}", pulsars(EDGE4, 81)), tm=True)
        T = fac * array_tspan(e.b)
        return e.curn(16, Tspan=T).fp(Tspan=T)
    R["tspan_0.5"] = lambda: tspan(0.5)
    R["tspan_2"] = lambda: tspan(2.0)

    # 9. geometry: near-coincident pulsars (HD, dipole, OS), sky points on a pulsar's line of sight (Fe, radiometer),
    # a 2-pulsar Fe array, a rank-deficient PSD ORF
    def coincident(orf):
        pos = [(5.0, 20.0), (5.0, 20.0 + math.degrees(1e-6)), (13.0, -35.0), (19.0, 60.0)]
        return _noise(Edge(f"coincident_{orf}", pulsars(EDGE4, 91, pos=pos)), tm=True).curn(1, hd=orf)
    R["coincident_hd"] = lambda: coincident("hd")
    R["coincident_dipole"] = lambda: coincident("dipole")

    def coincident_os():
        pos = [(5.0, 20.0), (5.0, 20.0 + math.degrees(1e-6)), (13.0, -35.0), (19.0, 60.0)]
        return _noise(Edge("coincident_os", pulsars(EDGE4, 92, pos=pos)), tm=True).os(8, orfs=("hd",))
    R["coincident_os"] = coincident_os

    def pole(P, inside=True):
        e = _noise(Edge(f"pole_{P}psr", pulsars(EDGE4[-P:], 93)), tm=True)
        sky = [near_pole_sky(e.b, 0, 2.0e-6), [[1.1, 2.2]]] + ([near_pole_sky(e.b, 0, 1.0e-6)] if inside else [])
        e.fp(n_freqs=2, sky=np.concatenate(sky))
        if P > 2:
            e.os(4, orfs=("hd",), lmax=None, sky=np.concatenate([near_pole_sky(e.b, 1, 1.0e-6), near_pole_sky(e.b, 1, 2.0e-6),
                                                   [[0.7, 3.3]]]))
        return e
    R["pole_4psr"] = lambda: pole(4)
    R["pole_2psr"] = lambda: pole(2, inside=False)

    def rank_psd():
        e = _noise(Edge("orf_rank2", pulsars(EDGE4, 94)), tm=True)
        v = np.array([[1.0, 0.6, -0.3, 0.2], [0.0, 0.8, 0.5, -0.9]])
        G = v.T @ v
        return e.curn(1, hd=G)
    R["orf_rank2"] = rank_psd

    def aniso():
        e = _noise(Edge("aniso_lmax1", pulsars((5, 7, 65, 193, 30, 40), 95)), tm=True)
        return e.os(4, orfs=("hd",), lmax=1, sky=[[0.4, 0.2], [2.0, 3.0]])
    R["aniso_lmax1"] = aniso

    # 10. chromatic noise: DM (idx 2) and scattering (idx 4) processes in every statistic's P_a
    def chrom_all():
        e = _noise(Edge("chrom_all", pulsars(EDGE4, 101, radio=True)), red=(-14.0, 4.0, 8))
        for i in range(e.b.n_psr):
            e.dm(i, -13.3, 2.5, 8)
            if e.b.ntoa[i] >= 20:
                e.chrom(i, -13.8, 3.0, 5)
                e.timing_model(i, poly=2, jumps="f", dm=1)
        return e.curn(4, hd="hd").os(4, orfs=("hd", "monopole")).pfos().fp(n_freqs=3, sky=[[0.4, 1.2], [2.2, 4.4]]).rn(4)
    R["chrom_all"] = chrom_all

    def chrom_single_freq():
        # pulsar 2 observes at 820 MHz only, with loud red and DM noise on the same frequencies: its two T blocks are
        # scaled copies and S is regularised only by Phi^-1
        e = _noise(Edge("chrom_single_freq", pulsars(EDGE4, 102, radio=True, single=(2,))), red=(-12.5, 3.0, 8), tm=True)
        for i in range(e.b.n_psr):
            e.dm(i, -12.3, 3.0, 8)
        return e.curn(4).os(4, orfs=("hd",)).pfos().fp(n_freqs=3).rn(4)
    R["chrom_single_freq"] = chrom_single_freq

    def chrom_dm_only_rn():
        # DM noise, no red noise: the red-noise likelihood leaves only the pulsar's own red noise out of P_a
        e = _noise(Edge("chrom_dm_only_rn", pulsars(EDGE4, 103, radio=True)), tm=True)
        for i in range(e.b.n_psr):
            e.dm(i, -12.8, 2.0, 8)
        return e.rn(4).curn(4)
    R["chrom_dm_only_rn"] = chrom_dm_only_rn

    def chrom_gw_modes():
        # loud DM noise exactly on the GW basis frequencies
        e = _noise(Edge("chrom_gw_modes", pulsars(EDGE4, 104, radio=True)), tm=True)
        T = array_tspan(e.b)
        for i in range(e.b.n_psr):
            e.dm(i, -12.0, 3.0, 4, modes=np.arange(1, 5) / T)
        return e.curn(4).os(4, orfs=("hd", "dipole")).pfos()
    R["chrom_gw_modes"] = chrom_gw_modes

    # 11. the red-noise likelihood's own: a pulsar spanning 3 days (a tiny T_a), and one Tspan for every pulsar
    R["rn_short_span"] = lambda: _noise(Edge("rn_short_span", pulsars((5, 24, 65), 111, spans={1: (55000.0, 55003.0)})),
                                        red=(-13.0, 3.0, 6)).rn(4)

    def rn_tspan():
        e = _noise(Edge("rn_tspan", pulsars(EDGE4, 112)), red=(-13.0, 3.0, 6), tm=True)
        return e.rn(4, Tspan=1.5 * array_tspan(e.b))
    R["rn_tspan"] = rn_tspan
    R["rn_common"] = lambda: _noise(Edge("rn_common", pulsars(EDGE4, 113)), red=(-13.0, 3.0, 6), tm=True).rn(
        4, log10_A_common=-13.5, gamma_common=3.0, components_common=6)
    return R


def collinear(accept):
    """4 pulsars, the two of at least 20 TOAs with a timing model that carries an extra column sin(2 pi t / Tspan + 1e-7) (table order), nearly the 1 /
    Tspan sine of the Fp basis.  ``accept``: Fp at frequencies far enough from 1 / Tspan that M_a(f) stays safely
    positive definite (1.2 / Tspan, 3 / Tspan); else at 1 / Tspan itself, which the timing model absorbs."""
    e = Edge("tm_collinear" if accept else "tm_collinear_refused", pulsars(EDGE4, 52))
    b = e.b
    T = array_tspan(b)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.1, log10_equad=-6.5)
        t = np.asarray(b.psrs[i].toas.table["tdbld"], dtype=float) * 86400.0
        if b.ntoa[i] >= 20:
            e.timing_model(i, poly=2, extra=np.sin(2 * np.pi * t / T + 1e-7))
    return e.fp(freqs=[1.2 / T, 3.0 / T] if accept else [1.0 / T, 3.0 / T])
