"""TEST INFRASTRUCTURE ONLY -- extended-precision reference of the summary kernels: the small reductions that turn a
map into the numbers a user reads (``curn_reduce_kernel``, ``fp_reduce_kernel`` + ``fp_q_int``, ``fe_combine_kernel``,
``os_aniso_reduce_kernel``, ``os_null_count_kernel``), and the constructed inputs the CPU and GPU tests share.

An independent restatement of what include/ptar.h promises, in ``np.longdouble`` (64-bit mantissa: ``RR.LONG``) with
``mpmath`` for Q(P, x).  Every floating-point output comes back as ``dict(hi, lo, bound, terms)`` for
``reduction_reference.check``.

Bounds of ``curn_summaries``.  With u = 2^-53 and eta = 2^-1074, the device's e = exp(fl(lnL - m)) carries the
subtraction's rounding through exp (relative |lnL - m| u), exp's own error (CUDA documents 1 ulp = 2 u for ``exp`` and
``log`` in double precision) and, where e is subnormal, an absolute eta:  |de| <= e (|lnL - m| + 3) u + 2 eta.  All sums
are of non-negative terms, so an n-term sum in any order adds gamma(n + 1) of itself; each product or quotient adds u.
``log10_A_ul`` inverts the trapezoid CDF: its bound is (CDF bound + target bound) / (mass of the interval) times the
interval's width, and where those bounds let the target fall on either side of a node both neighbouring intervals are
acceptable (as ``exceed_lo`` / ``exceed_hi`` of ``reduction_reference.os_null``): the acceptable set is the hull of the
candidate intervals' ranges, returned as its midpoint and half-width.

The non-finite rule (include/ptar.h): every (max, argmax) ranks by larger value, then lower index, the first NaN above
every number (``first_max``); a map with a NaN or +inf has NaN integrals; an all -inf map has ln_bayes = -inf and NaN
posteriors; -inf among finite entries is an ordinary zero.

``mutant=`` selects a deliberately wrong variant (``CURN_MUTANTS``, ``FP_MUTANTS``, ``MAX_MUTANTS``) so that the CPU
test can show that the constructed cases reject each of them.  Two tempting mutants are absent because they compute
the same function: a CDF normalised by 1 instead of its last node (the last node is sum_k wx_k post_k = 1 by the
normalisation of the posterior), and fp_q_int's m switched at x = P instead of P - 1 (floor x = P - 1 on [P - 1, P)
either way); ``m_switch_late`` switches one integer later, where the sum gains a term."""
from __future__ import annotations

import numpy as np

from tests import reduction_reference as RR

U = RR.U
ETA = 2.0 ** -1074
LD = np.longdouble
EXP_ULP = 2.0          # assumed device error of exp and log, in units of u (1 ulp)

MAX_MUTANTS = ("tie_high", "max_skips_nan", "max_last_nan")
CURN_MUTANTS = ("amp_major", "no_prior", "end_weight", "cdf_end_weight", "ul_wrong_end")
FP_MUTANTS = ("q_term_few", "q_term_many", "m_switch_late")


def _out(h, bound, terms=None):
    """check dict of a longdouble array: hi + lo and the bound plus the reference's own rounding."""
    h = np.asarray(h, dtype=LD)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = h.astype(np.float64)
        lo = np.where(np.isfinite(hi), (h - hi.astype(LD)), 0).astype(np.float64)
    return dict(hi=hi, lo=lo, bound=np.asarray(bound, dtype=np.float64), terms=np.abs(hi) if terms is None else terms)


# ------------------------------------------------------------------ the one (max, argmax) rule
def first_max(values, mutant=None):
    """Index of the maximum of a 1-D array: larger value, then lower index, the first NaN above every number."""
    v = np.asarray(values, dtype=np.float64).ravel()
    nan = np.flatnonzero(np.isnan(v))
    if nan.size and mutant != "max_skips_nan":
        return int(nan[-1] if mutant == "max_last_nan" else nan[0])
    if nan.size == v.size:
        return 0
    m = np.nanmax(v)
    hit = np.flatnonzero(v == m)
    return int(hit[-1] if mutant == "tie_high" else hit[0])


# ------------------------------------------------------------------ grids, weights, priors (restated)
def trapezoid_weights(v):
    """Trapezoid weights of increasing nodes in longdouble: half the neighbouring intervals, 1 for a single node."""
    v = np.asarray(v, dtype=np.float64).astype(LD)
    if v.size == 1:
        return np.ones(1, dtype=LD)
    d = np.diff(v)
    w = np.zeros(v.size, dtype=LD)
    w[:-1] += d / 2
    w[1:] += d / 2
    return w


def prior_density(log10_A, gamma, kind):
    """Prior density per log10 A on the nodes, longdouble: constant ("log-uniform") or proportional to A = 10^x
    ("uniform" in A), normalised so that sum_g sum_k wg wx prior = 1."""
    x = np.asarray(log10_A, dtype=np.float64).astype(LD)
    if kind == "log-uniform":
        p = np.ones(x.size, dtype=LD)
    elif kind == "uniform":
        p = np.exp((x - x[-1]) * np.log(LD(10)))
    else:
        raise ValueError(kind)
    return p / (trapezoid_weights(gamma).sum() * np.sum(trapezoid_weights(x) * p))


def statics(log10_A, gamma, kind):
    """The fp64 statics a ptar_curn_model holds for this grid: dict log10_A, gamma, wg, wx, prior."""
    f = lambda a: np.asarray(a, dtype=LD).astype(np.float64)
    return dict(log10_A=f(log10_A), gamma=f(gamma), wg=f(trapezoid_weights(gamma)), wx=f(trapezoid_weights(log10_A)),
                prior=f(prior_density(log10_A, gamma, kind)))


def nodes(n, spacing, lo, step):
    """n increasing nodes from ``lo``: "uniform" (step a power of two, so sums of intervals are exact), "geometric"
    (intervals growing by 2 % each) or "tiny" (uniform with the middle interval 1e-9)."""
    if n == 1:
        return np.array([lo + 2.0])
    d = np.full(n - 1, float(step))
    if spacing == "geometric":
        d = step * 1.02 ** np.arange(n - 1)
    elif spacing == "tiny":
        d[(n - 1) // 2] = 1e-9
    elif spacing != "uniform":
        raise ValueError(spacing)
    return lo + np.r_[0.0, np.cumsum(d)]


GRIDS = ((2, 1), (3, 2), (255, 1), (256, 256), (64, 5), (97, 57))      # (NA, NG)
SPACINGS = ("uniform", "geometric", "tiny")
PRIORS = ("log-uniform", "uniform")
ULS = (1e-6, 0.5, 0.95, 1 - 1e-12)


def grid(NA, NG, spacing):
    return nodes(NA, spacing, -18.0, 2.0 ** -5), nodes(NG, spacing, 0.0, 2.0 ** -6)


# ------------------------------------------------------------------ CURN summaries
def curn_core(lnL, log10_A, gamma, wg, wx, prior, mutant=None):
    """Everything of ``curn_summaries`` but the upper limit; ``lnL`` [R, NG, NA]."""
    assert RR.LONG, "the reference needs a 64-bit mantissa longdouble"
    lnL = np.asarray(lnL, dtype=np.float64)
    R, NG, NA = lnL.shape
    x = np.asarray(log10_A, dtype=np.float64)
    wgl, wxl, pl = (np.asarray(v, dtype=np.float64).astype(LD) for v in (wg, wx, prior))
    if mutant == "end_weight" and NA > 1:
        wxl = wxl.copy()
        wxl[0], wxl[-1] = 2 * wxl[0], 2 * wxl[-1]
    flat = lnL.transpose(0, 2, 1).reshape(R, -1) if mutant == "amp_major" else lnL.reshape(R, -1)
    am = np.array([first_max(flat[r], mutant) for r in range(R)])
    m = flat[np.arange(R), am]
    if mutant == "amp_major":
        ig, ia = am % NG, am // NG
    else:
        ig, ia = am // NA, am % NA
    with np.errstate(invalid="ignore", over="ignore", under="ignore", divide="ignore"):
        bad = ~(np.isfinite(m)) | np.isposinf(lnL).any(axis=(1, 2)) | np.isnan(lnL).any(axis=(1, 2))
        ms = np.where(bad, 0.0, m)
        d = lnL.astype(LD) - ms.astype(LD)[:, None, None]
        e = np.where(np.isneginf(lnL), LD(0), np.exp(np.where(np.isfinite(d), d, 0)))
        ad = np.where(np.isfinite(d), np.abs(d), 0).astype(np.float64)
        eb = e.astype(np.float64) * (ad + 1 + EXP_ULP) * U + 2 * ETA                   # |de|
        wgf, wpf = wgl.astype(np.float64), (wxl * pl).astype(np.float64)
        S = np.einsum("g,rgk->rk", wgl, e)
        Sb = np.einsum("g,rgk->rk", wgf, eb) + RR.gamma(NG + 1) * S.astype(np.float64) + NG * ETA
        T = np.einsum("k,rgk->rg", wxl * pl, e)
        Tb = np.einsum("k,rgk->rg", wpf, eb) + RR.gamma(NA + 3) * T.astype(np.float64) + NA * ETA
        B = S @ (wxl * pl)
        Bf = B.astype(np.float64)
        Bb = Sb @ wpf + RR.gamma(NA + 11) * Bf + NA * ETA
        lnB = np.log(B)
        lnb = ms.astype(LD) + lnB
        lnbb = Bb / Bf + EXP_ULP * U * np.abs(lnB.astype(np.float64)) + U * np.abs(lnb.astype(np.float64))
        pa = (S if mutant == "no_prior" else pl[None, :] * S) / B[:, None]
        paf = pa.astype(np.float64)
        pab = pl.astype(np.float64)[None, :] * Sb / Bf[:, None] + paf * (Bb / Bf + 3 * U)[:, None] + 2 * ETA * (1 + 1 / Bf)[:, None]
        pg = T / B[:, None]
        pgf = pg.astype(np.float64)
        pgb = Tb / Bf[:, None] + pgf * (Bb / Bf + 2 * U)[:, None] + 2 * ETA * (1 + 1 / Bf)[:, None]
    nan = np.full(R, np.nan)
    lnb = np.where(bad, np.where(np.isneginf(m), -np.inf, nan).astype(LD), lnb)
    lnbb = np.where(bad, 0.0, lnbb)
    pa, pab = np.where(bad[:, None], LD(np.nan), pa), np.where(bad[:, None], 0.0, pab)
    pg, pgb = np.where(bad[:, None], LD(np.nan), pg), np.where(bad[:, None], 0.0, pgb)
    return dict(lnL_max=m, ml_gamma_index=ig, ml_log10_A_index=ia, ln_bayes=_out(lnb, lnbb),
                post_log10_A=_out(pa, pab), post_gamma=_out(pg, pgb), _pa=pa, _pab=pab, _x=x, _bad=bad, _mutant=mutant)


def curn_ul(core, ul):
    """log10_A_ul [R] of a ``curn_core`` result: the quantile ``ul`` of the trapezoid CDF of post_log10_A, normalised
    by its last node, linear between nodes; the hull of every interval the bounds admit (module docstring)."""
    pa, pab, x, mutant = core["_pa"], core["_pab"], core["_x"], core["_mutant"]
    R, NA = pa.shape
    dx = np.diff(x.astype(LD))
    mid, half = np.full(R, np.nan), np.zeros(R)
    for r in np.flatnonzero(~core["_bad"]):
        w = 0.5 * dx * (pa[r, 1:] + pa[r, :-1])
        if mutant == "cdf_end_weight":
            w = w.copy()
            w[0] += 0.5 * dx[0] * pa[r, 0]
            w[-1] += 0.5 * dx[-1] * pa[r, -1]
        C = np.r_[LD(0), np.cumsum(w)]
        wb = 0.5 * dx.astype(np.float64) * (pab[r, 1:] + pab[r, :-1])
        Cb = np.r_[0.0, np.cumsum(wb)] + RR.gamma(np.arange(NA) + 4) * C.astype(np.float64) + np.arange(NA) * ETA
        t = LD(ul) * C[-1]
        tb = float(ul) * Cb[-1] + U * float(t)
        s = tb + Cb[1:] + Cb[:-1]                                               # per interval k = 1 .. NA - 1
        cand = np.flatnonzero((C[:-1].astype(np.float64) - s <= float(t)) & (float(t) <= C[1:].astype(np.float64) + s))
        if cand.size == 0:                                                      # a mutant's target beyond the CDF
            cand = np.array([NA - 2])
        lo, hi = np.inf, -np.inf
        for k in cand:
            mass = float(w[k])
            f = float(np.clip((t - C[k]) / w[k], 0, 1)) if mass > 0 else 0.0
            if mutant == "ul_wrong_end":
                f = 1.0 - f
            df = 2.2 * s[k] / mass if mass > 0 else 1.0
            df = 1.0 if df > 0.1 else df
            slack = 4 * U * max(abs(x[k]), abs(x[k + 1]))
            lo = min(lo, x[k] + float(dx[k]) * max(0.0, f - df) - slack)
            hi = max(hi, x[k] + float(dx[k]) * min(1.0, f + df) + slack)
        mid[r], half[r] = 0.5 * (lo + hi), 0.5 * (hi - lo) * (1 + 4 * U)
    return dict(hi=mid, lo=np.zeros(R), bound=half, terms=np.abs(mid))


def curn_summaries(lnL, log10_A, gamma, wg, wx, prior, ul, mutant=None):
    """Reference of ptar_curn_reduce on maps ``lnL`` [R, NG, NA] with the fp64 statics the model holds: lnL_max and
    the first gamma-major argmax (exact), ln_bayes, post_log10_A, post_gamma, log10_A_ul (check dicts)."""
    core = curn_core(lnL, log10_A, gamma, wg, wx, prior, mutant)
    out = {k: v for k, v in core.items() if not k.startswith("_")}
    out["log10_A_ul"] = curn_ul(core, ul)
    return out


def check(dev, ref, what="", report=None, family=None):
    """``RR.check`` where the reference is finite; where it is NaN or infinite the device must hold the same."""
    dev = np.asarray(dev, dtype=np.float64)
    nf = ~np.isfinite(ref["hi"])
    assert np.array_equal(dev[nf], ref["hi"][nf], equal_nan=True), \
        f"{what}: non-finite outputs differ: device {dev[nf]}, reference {ref['hi'][nf]}"
    rk = dict(ref, hi=np.where(nf, 0.0, ref["hi"]), lo=np.where(nf, 0.0, ref["lo"]))
    return RR.check(np.where(nf, 0.0, dev), rk, what, report, family)


CURN_EXACT = ("lnL_max", "ml_gamma_index", "ml_log10_A_index")
CURN_BOUNDED = ("ln_bayes", "post_log10_A", "post_gamma", "log10_A_ul")


def curn_compare(dev, ref, what="", report=None, family="curn_reduce", slack=0.0):
    """``dev`` (dict of numpy arrays with the keys of ``curn_summaries``) against ``ref``; ``slack`` widens each
    relative bound by that many u (an fp64 oracle that rounds its own statics).  Returns the worst |d| / bound."""
    for k in CURN_EXACT:
        assert np.array_equal(np.asarray(dev[k]), np.asarray(ref[k]), equal_nan=True), \
            f"{what} {k}: {np.asarray(dev[k])} != {np.asarray(ref[k])}"
    worst = 0.0
    for k in CURN_BOUNDED:
        rk = dict(ref[k])
        rk["bound"] = rk["bound"] + slack * U * np.abs(np.nan_to_num(rk["hi"], posinf=0, neginf=0))
        worst = max(worst, check(dev[k], rk, f"{what} {k}", report, family)[0])
    return worst


# ------------------------------------------------------------------ constructed maps
def ridge(x, g, height=30.0):
    """A smooth Gaussian ridge peaking inside the grid: the ordinary map."""
    xs = (x - x[0]) / max(x[-1] - x[0], 1e-300)
    gs = (g - g[0]) / max(g[-1] - g[0], 1e-300) if g.size > 1 else np.zeros(1)
    return height * (-0.5 * ((xs[None, :] - 0.6) / 0.08) ** 2 - 0.5 * ((gs[:, None] - 0.4) / 0.2) ** 2)


FLOORS = (30.0, 700.0, 745.0, 1e4, np.inf)


def spike_sites(NA, NG):
    s = [(0, 0), (0, NA - 1), (NG - 1, 0), (NG - 1, NA - 1), (NG // 2, 0), (NG // 2, NA - 1), (NG // 2, NA // 2)]
    return list(dict.fromkeys(s))


def tie_sites(n):
    """Flat-index pairs that hold the repeated maximum: the same reduce thread's stride (e, e + 256), different
    threads, different halves of the 256-thread tree, and with the winner not the first entry of its thread."""
    pairs = [(5, 261), (261, 517), (3, 200), (130, 263), (n - 2, n - 1), (0, n - 1), (127, 128), (300, 44)]
    return [tuple(sorted(p)) for p in dict.fromkeys(pairs) if max(p) < n and p[0] != p[1] and min(p) >= 0]


def curn_maps(x, g, seed=0):
    """(names, maps [R, NG, NA]) of the finite and -inf families on the grid (x, g)."""
    NA, NG = x.size, g.size
    n = NA * NG
    rng = np.random.default_rng(seed + n)
    names, maps = [], []

    def add(name, m):
        names.append(name)
        maps.append(np.asarray(m, dtype=np.float64).reshape(NG, NA))

    for c in (0.0, 3.5, 1e300, -1e300):
        add(f"const {c:g}", np.full(n, c))
    rd = ridge(x, g)
    add("ridge", rd)
    base = -1.0 - rng.uniform(0, 5, n)
    for a, c in tie_sites(n):
        m = base.copy()
        m[[a, c]] = 2.0
        add(f"tie {a},{c}", m)
    for (sg, sk) in spike_sites(NA, NG):
        for fl in FLOORS:
            m = np.full((NG, NA), 12.25 - fl)                                    # lnL - m = -fl exactly
            m[sg, sk] = 12.25
            add(f"spike g{sg} k{sk} floor {fl:g}", m)
    if NA >= 8:
        for fl in (1e4, np.inf):
            m = np.full((NG, NA), 7.0 - fl)
            m[NG // 2, 2] = m[NG // 2, NA - 3] = 7.0
            add(f"two spikes floor {fl:g}", m)
    m = rd.copy().ravel()
    m[rng.random(n) < 0.1] = -np.inf
    m[int(np.argmax(rd))] = rd.max()
    add("ridge with -inf holes", m)
    return names, np.stack(maps)


NONFINITE = (np.nan, np.inf, -np.inf)


def positions(n):
    """First, last, index 128 and the middle of an axis of length n (deduplicated, in range)."""
    return [p for p in dict.fromkeys((0, n - 1, 128, n // 2)) if 0 <= p < n]


def curn_nonfinite_maps(x, g):
    """(names, maps): a ridge with one NaN / +inf / -inf at each of ``positions``, NaN together with +inf, two NaNs,
    and the all -inf map."""
    NA, NG = x.size, g.size
    n = NA * NG
    rd = ridge(x, g).ravel()
    names, maps = [], []
    for v in NONFINITE:
        for p in positions(n):
            m = rd.copy()
            m[p] = v
            names.append(f"{v} at {p}")
            maps.append(m)
    p = positions(n)
    m = rd.copy()
    m[p[0]], m[p[-1]] = np.inf, np.nan
    names.append("+inf before NaN")
    maps.append(m)
    m = rd.copy()
    m[p[-1]] = m[p[1]] = np.nan
    names.append("two NaN")
    maps.append(m)
    names.append("all -inf")
    maps.append(np.full(n, -np.inf))
    return names, np.stack(maps).reshape(-1, NG, NA)


# ------------------------------------------------------------------ Fp summaries
Q_CONST = 4.0          # |dQ| <= Q_CONST (x + P) u Q + 4 eta: the header's "(Fp + n_psr) 2^-53" with its constant


def q_ref(P, x, mutant=None):
    """Q(P, x) = Gamma(P, x) / Gamma(P) of fp64 x >= 0 (array) by mpmath at 60 digits: (longdouble values, bound).
    Values below the longdouble range come back as 0.  NaN stays NaN."""
    import mpmath
    xfull = np.atleast_1d(np.asarray(x, dtype=np.float64))
    x, inverse = np.unique(xfull.ravel(), return_inverse=True)               # NaNs collapse to one
    out = np.empty(x.shape, dtype=LD)
    with mpmath.workdps(60):
        for i, v in np.ndenumerate(x):
            if np.isnan(v):
                out[i] = np.nan
            elif np.isinf(v):
                out[i] = 0
            elif mutant is None:
                q = mpmath.gammainc(P, mpmath.mpf(float(v)), mpmath.inf, regularized=True) if v > 0 else mpmath.mpf(1)
                out[i] = _ld_of_mpf(q)
            else:
                nt = P - 1 if mutant == "q_term_few" else P + 1 if mutant == "q_term_many" else \
                    (P + 1 if P <= v < P + 1 else P)                           # m_switch_late: floor(x) = P is used
                xv = mpmath.mpf(float(v))
                q = mpmath.exp(-xv) * mpmath.fsum(xv ** k / mpmath.factorial(k) for k in range(nt))
                out[i] = _ld_of_mpf(q)
    out, x = out[inverse].reshape(xfull.shape), xfull
    with np.errstate(invalid="ignore", over="ignore"):
        qf = out.astype(np.float64)
        bound = ((np.where(np.isfinite(x), x, 0.0) + P) * U) * qf * Q_CONST + 4 * ETA
    return out, np.where(np.isnan(bound), 0.0, bound)


def _ld_of_mpf(q):
    import mpmath
    if q < mpmath.mpf(2) ** -1100:
        return LD(0)
    hi = float(q)
    return LD(hi) + LD(float(q - mpmath.mpf(hi)))


def fp_summaries(amps, n_psr, mutant=None):
    """Reference of ptar_fp_reduce_fap on ``amps`` [R, P, 2 Nf]: Fp (pulsar order; check dict), Fp_max and the first
    argmax of the fp64 Fp (exact where Fp is exactly representable, as the constructed cases make it), fap =
    Q(P, Fp) of that fp64 Fp (check dict)."""
    assert RR.LONG
    a = np.asarray(amps, dtype=np.float64)
    R, P, nc = a.shape
    assert P == n_psr
    with np.errstate(invalid="ignore", over="ignore"):
        al = a.astype(LD).reshape(R, P, nc // 2, 2)
        F = (al * al).sum(axis=(1, 3)) / 2                                       # [R, Nf]
        Ff = F.astype(np.float64)
        Fb = RR.gamma(2 * P + 2) * np.where(np.isfinite(Ff), Ff, 0.0) + 4 * ETA
    am = np.array([first_max(Ff[r], mutant) for r in range(R)])
    q, qb = q_ref(P, Ff, mutant)
    return dict(Fp=_out(F, Fb), Fp_max=Ff[np.arange(R), am], Fp_argmax=am, fap=_out(q, qb))


def fp_x_values(P):
    """The sweep of Fp values x for n_psr = P: both sides of every branch of fp_q_int (m = 0, the exact-factorial
    branch, Stirling from m = 16, m = floor x -> P - 1 at x = P - 1), integers +- 1 ulp, the tails down to underflow."""
    xs = [0.0, 5e-324, 1e-300, 0.5, np.nextafter(1.0, 0), 1.0]
    for c in (15.0, 16.0, float(P - 1)):
        if c > 0:
            xs += [np.nextafter(c, 0), c, np.nextafter(c, np.inf)]
    xs += [float(P), 10.0 * P, 700.0, 745.0, 1e4, 8e307, np.inf]             # Fp = 1/2 s <= DBL_MAX / 2
    return np.array(list(dict.fromkeys(xs)))


def exact_pair(x):
    """(a, b) with 1/2 fl(b b + fl(a a)) == x, the expression of fp_reduce_kernel for one pulsar: a = sqrt(2 x) cut to
    26 bits (its square is exact), b = sqrt of the remainder (its square's rounding is far below half an ulp of 2 x).
    x = inf -> (1e200, 0).  Verified here in exact rational arithmetic."""
    from fractions import Fraction
    import math
    if np.isinf(x):
        return 1e200, 0.0
    t = 2.0 * x
    assert np.isfinite(t), "Fp = 1/2 s: values above DBL_MAX / 2 are not reachable"
    mant, ex = math.frexp(math.sqrt(t))
    a = math.ldexp(math.floor(mant * 2.0 ** 26), ex - 26)
    b = math.sqrt(max(t - a * a, 0.0))
    assert 0.5 * float(Fraction(a * a) + Fraction(b) ** 2) == x, x
    return a, b


def fp_amps_of(xs, P, Nf, split=False):
    """amps [R, P, 2 Nf] whose Fp[r][f] is exactly xs[(r + f) % len(xs)]: pulsar (r + f) mod P carries ``exact_pair``,
    the others 0.  ``split`` instead gives every pulsar (sqrt(2 x / P), 0): Fp = x up to rounding, every pulsar in
    the sum."""
    R = len(xs)
    a = np.zeros((R, P, 2 * Nf))
    for r in range(R):
        for f in range(Nf):
            x = xs[(r + f) % R]
            if split:
                a[r, :, 2 * f] = np.sqrt(2 * x / P) if np.isfinite(x) else 1e200
            else:
                a[r, (r + f) % P, 2 * f:2 * f + 2] = exact_pair(x)
    return a


# ------------------------------------------------------------------ the small combines
def fe_combine(fmax, fargmax, mutant=None):
    """Reference of ptar_fe_combine: fe_max, argmax_f (``first_max`` over f), argmax_sky = fargmax of the winner."""
    fmax = np.asarray(fmax, dtype=np.float64)
    am = np.array([first_max(row, mutant) for row in fmax])
    r = np.arange(len(fmax))
    return dict(fe_max=fmax[r, am], argmax_f=am, argmax_sky=np.asarray(fargmax)[r, am])


def null_count(snr):
    """Reference of os_null_count: null_exceed = #{s >= 1 : not S/N_s < S/N_0} (a NaN null column counts), fap =
    (1 + null_exceed) / n_col, NaN when S/N_0 is NaN."""
    snr = np.asarray(snr, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        ex = np.sum(~(snr[:, 1:] < snr[:, :1]), axis=1)
    fap = np.where(np.isnan(snr[:, 0]), np.nan, (1.0 + ex) / snr.shape[1])
    return dict(null_exceed=ex, fap=fap)
