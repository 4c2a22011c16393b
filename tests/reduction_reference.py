"""Extended-precision reference of the per-realization reductions (timing fit, optimal statistic, its null
distributions, Fp-statistic) with a rigorous componentwise error bound per output -- numpy only, no torch.

The reference evaluates exactly the operation the kernels evaluate, on the fp64 statics the device holds (pulled back
from ``compile()``), so only the kernels' arithmetic is under test.  Values are carried as unevaluated pairs hi + lo
of fp64 numbers: dot products run in ``np.longdouble`` where it has a 64-bit mantissa and as Ogita-Rump-Oishi Dot2
(error-free TwoProduct / TwoSum) elsewhere; scalings and divisions by fp64 statics are error-free transformations.

Bounds.  A projection y = sum_i a_i b_i over n terms, summed in any order (tensor-core fragments, k-splits, tile sums,
alignment zeros), satisfies |dy| <= gamma_{n+8} sum_i |a_i b_i|, gamma_m = m u / (1 - m u), u = 2^-53.  Later stages
propagate it to first order and add their own rounding: x = X phi~^1/2, d_ab = x_a . x_b, rho = d / t, the template sums
b, A^2 = b / D, S/N = b / sqrt(D), F^-1 b; U . V / sqrt(D_s) for the null; Fp = 1/2 sum_a |X^_a|^2; and
r' = r - W^-1/2 Q (Q^T W^1/2 r) including the s_i r_i products and the 1/sqrt(w) division.  The bounds hold for any
summation order, so they stay valid under a rewrite of a kernel's reduction tree and where outputs cancel.

``check`` reports, per output, the worst |d| / bound (must be <= 1) and the worst |d| / (u sum|terms|) (information).
``q_int`` is Q(P, x) = Gamma(P, x) / Gamma(P) for integer P, the algorithm of ``fp_q_int`` in csrc/ptar_fp.cuh.

The second half builds the edge batches (TOA counts, basis widths, templates, timing models) that the CPU and GPU
tests share."""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -53
LONG = np.finfo(np.longdouble).nmant >= 63
LD = np.longdouble


def gamma(m):
    m = np.asarray(m, dtype=float)
    return m * U / (1.0 - m * U)


# ------------------------------------------------------------------ error-free transformations
def two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fast_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


def _split(a):
    c = 134217729.0 * a
    h = c - (c - a)
    return h, a - h


def two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _pair_of_ld(v):
    hi = v.astype(np.float64)
    return hi, (v - hi.astype(LD)).astype(np.float64)


def xmatmul(A, B, dot2=None):
    """A [.., m, n] @ B [n, c] (fp64 inputs) in twice the working precision: (hi, lo)."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    if (LONG if dot2 is None else not dot2):
        return _pair_of_ld(A.astype(LD) @ B.astype(LD))
    s = np.zeros(A.shape[:-1] + B.shape[-1:])
    err = np.zeros_like(s)
    for i in range(A.shape[-1]):
        p, e = two_prod(A[..., i:i + 1], B[i:i + 1, :])
        s, q = two_sum(s, p)
        err += q + e
    return fast_two_sum(s, err)


def xsum_prod(ah, al, bh, bl, axis=-1, dot2=None):
    """sum over ``axis`` of (ah + al)(bh + bl), broadcasting, in twice the working precision: (hi, lo)."""
    if (LONG if dot2 is None else not dot2):
        return _pair_of_ld(((np.asarray(ah).astype(LD) + al) * (np.asarray(bh).astype(LD) + bl)).sum(axis=axis))
    ah, al, bh, bl = (np.moveaxis(v, axis, 0) for v in np.broadcast_arrays(*(np.asarray(v, dtype=np.float64)
                                                                            for v in (ah, al, bh, bl))))
    s = np.zeros(ah.shape[1:])
    err = np.zeros_like(s)
    for i in range(ah.shape[0]):
        p, e = two_prod(ah[i], bh[i])
        s, q = two_sum(s, p)
        err += q + e + (ah[i] * bl[i] + al[i] * bh[i])
    return fast_two_sum(s, err)


def xscale(h, l, s):
    """(h + l) * s, s fp64."""
    p, e = two_prod(h, s)
    return fast_two_sum(p, e + l * s)


def xdiv(h, l, t):
    """(h + l) / t, t fp64."""
    q = h / t
    p, e = two_prod(q, t)
    return fast_two_sum(q, ((h - p) - e + l) / t)


def xsub(a, h, l):
    """a - (h + l), a fp64."""
    s, e = two_sum(a, -h)
    return fast_two_sum(s, e - l)


# ------------------------------------------------------------------ checking
class Report:
    """Worst |d| / bound and |d| / (u sum|terms|) per kernel family."""

    def __init__(self):
        self.worst = {}

    def add(self, family, ratio, info):
        w = self.worst.setdefault(family, [0.0, 0.0])
        w[0], w[1] = max(w[0], ratio), max(w[1], info)

    def lines(self):
        return [f"{k:>12s}: worst |d|/bound {v[0]:.3f}, worst |d|/(u sum|terms|) {v[1]:.3f}" for k, v in sorted(self.worst.items())]


def check(dev, ref, what="", report=None, family=None):
    """``dev`` (fp64 array) against ``ref`` = dict(hi, lo, bound, terms).  Returns (worst |d| / bound,
    worst |d| / (u terms)); raises AssertionError when an output is outside its bound."""
    dev = np.asarray(dev, dtype=np.float64)
    d = np.abs((dev - ref["hi"]) - ref["lo"])
    b, t = np.broadcast_to(ref["bound"], d.shape), np.broadcast_to(ref["terms"], d.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / b)
        i = np.where(d == 0, 0.0, d / (U * t))
    r = np.where(np.isnan(dev) != np.isnan(ref["hi"]), np.inf, np.nan_to_num(r, nan=np.inf))
    worst, info = (float(r.max()), float(np.nan_to_num(i, nan=np.inf, posinf=np.inf).max())) if r.size else (0.0, 0.0)
    if report is not None and family is not None:
        report.add(family, worst, info)
    if not worst <= 1.0:
        k = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError(f"{what}: |d| / bound = {worst:.3g} at {k}: device {dev[k]!r}, reference {ref['hi'][k]!r} "
                             f"+ {ref['lo'][k]!r}, bound {b[k]:.3e}")
    return worst, info


def _out(h, l, bound, terms):
    return dict(hi=h, lo=l, bound=bound, terms=terms)


# ------------------------------------------------------------------ reductions
def projection(rows, B, s, n, dot2=None):
    """y[r][j] = sum_{i < n} B[s + i][j] rows[r][s + i] (the TOAs of one pulsar): (hi, lo, bound, sum|terms|)."""
    A = rows[:, s:s + n]
    Bp = B[s:s + n]
    h, l = xmatmul(A, Bp, dot2)
    t = np.abs(A) @ np.abs(Bp)
    return h, l, gamma(n + 8) * t, t


def optimal_statistic(S, rows, dot2=None):
    """Reference of ptar_os_project + ptar_os_pairs.  ``S``: dict C [ld, ncp], nc, sqrt_phi [ncp], pairs [q, 2],
    t_ab, orf [n_orf, q], dnorm, dsqrt, finv [n_orf, n_orf], seg_off, seg_len (the device's statics).  Returns
    dict X, x (hi, lo, bound) and rho, A2, snr, A2_mc (check dicts)."""
    nc = S["nc"]
    R, P = rows.shape[0], len(S["seg_off"])
    Xh, Xl, XB, XT = (np.zeros((R, P, nc)) for _ in range(4))
    for a in range(P):
        Xh[:, a], Xl[:, a], XB[:, a], XT[:, a] = projection(rows, S["C"][:, :nc], S["seg_off"][a], S["seg_len"][a], dot2)
    sp = S["sqrt_phi"][:nc]
    xh, xl = xscale(Xh, Xl, sp)
    xb = XB * sp + U * np.abs(xh)
    xt = XT * sp                                  # sum|terms| propagated (information only)
    pa, pb = S["pairs"][:, 0], S["pairs"][:, 1]
    dh, dl = xsum_prod(xh[:, pa], xl[:, pa], xh[:, pb], xl[:, pb], dot2=dot2)
    db = np.sum(xb[:, pa] * np.abs(xh[:, pb]) + np.abs(xh[:, pa]) * xb[:, pb], axis=-1) + \
        gamma(nc) * np.sum(np.abs(xh[:, pa] * xh[:, pb]), axis=-1)
    dt = np.sum(xt[:, pa] * xt[:, pb], axis=-1)
    out = dict(X=(Xh, Xl, XB), x=(xh, xl, xb), xt=xt, d=(dh, dl, db), dt=dt)
    rh, rl = xdiv(dh, dl, S["t_ab"])
    out["rho"] = _out(rh, rl, db / S["t_ab"] + U * np.abs(rh), dt / S["t_ab"])
    W = S["orf"]
    nq = W.shape[1]
    bh, bl = xsum_prod(W[None], 0.0, dh[:, None, :], dl[:, None, :], dot2=dot2)          # [R, n_orf]
    bb = db @ np.abs(W).T + gamma(nq + 8) * (np.abs(dh) @ np.abs(W).T)
    bt = dt @ np.abs(W).T
    ah, al = xdiv(bh, bl, S["dnorm"])
    out["A2"] = _out(ah, al, bb / S["dnorm"] + U * np.abs(ah), bt / S["dnorm"])
    sh, sl = xdiv(bh, bl, S["dsqrt"])
    out["snr"] = _out(sh, sl, bb / S["dsqrt"] + U * np.abs(sh), bt / S["dsqrt"])
    Fi = S["finv"]
    mh, ml = xsum_prod(Fi[None], 0.0, bh[:, None, :], bl[:, None, :], dot2=dot2)
    out["A2_mc"] = _out(mh, ml, bb @ np.abs(Fi).T + gamma(Fi.shape[0]) * (np.abs(bh) @ np.abs(Fi).T), bt @ np.abs(Fi).T)
    return out


def os_null(S, N, osref, dot2=None):
    """Reference of ptar_os_null: S/N[r][s] = U[r] . V[:, s] / sqrt(D_s) and the counts.  ``N``: dict method,
    V [n_colp, kdp], kd, n_col, dsqrt [n_col].  Returns dict snr (check dict), and the bracket (lo, hi) of
    null_exceed that any result within the bounds must fall in."""
    xh, xl, xb = osref["x"]
    pa, pb = S["pairs"][:, 0], S["pairs"][:, 1]
    R, nq, nc = xh.shape[0], len(pa), S["nc"]
    if N["method"] == "phase_shift":
        K = nc // 2
        ah, al, ab = (v[:, pa].reshape(R, nq, K, 2) for v in (xh, xl, xb))
        bh, bl, bbb = (v[:, pb].reshape(R, nq, K, 2) for v in (xh, xl, xb))
        # (q, k, 0) = a0 b0 + a1 b1;  (q, k, 1) = a1 b0 - a0 b1
        Bh = np.stack([bh, np.stack([-bh[..., 1], bh[..., 0]], axis=-1)], axis=3)           # [R, q, K, 2(out), 2]
        Bl = np.stack([bl, np.stack([-bl[..., 1], bl[..., 0]], axis=-1)], axis=3)
        Bb = np.stack([bbb, bbb[..., ::-1]], axis=3)
        uh, ul = xsum_prod(ah[:, :, :, None, :], al[:, :, :, None, :], Bh, Bl, dot2=dot2)
        ub = np.sum(ab[:, :, :, None, :] * np.abs(Bh) + np.abs(ah[:, :, :, None, :]) * Bb, axis=-1) + \
            gamma(2) * np.sum(np.abs(ah[:, :, :, None, :] * Bh), axis=-1)
        at, bt = (osref["xt"][:, v].reshape(R, nq, K, 2) for v in (pa, pb))
        ut = np.sum(at[:, :, :, None, :] * np.stack([bt, bt[..., ::-1]], axis=3), axis=-1)
        uh, ul, ub, ut = (v.reshape(R, -1) for v in (uh, ul, ub, ut))
    else:
        uh, ul, ub = osref["d"]
        ut = osref["dt"]
    V = N["V"][:N["n_col"], :N["kd"]].T                                                   # [kd, n_col]
    nh, nl = xmatmul(uh, V, dot2)
    nl = nl + ul @ V
    nh, nl = fast_two_sum(nh, nl)
    nb = ub @ np.abs(V) + gamma(N["kd"] + 8) * (np.abs(uh) @ np.abs(V))
    nt = ut @ np.abs(V)
    sh, sl = xdiv(nh, nl, N["dsqrt"])
    snr = _out(sh, sl, nb / N["dsqrt"] + U * np.abs(sh), nt / N["dsqrt"])
    diff = (sh[:, 1:] - sh[:, :1]) + (sl[:, 1:] - sl[:, :1])
    tie = snr["bound"][:, 1:] + snr["bound"][:, :1]
    return dict(snr=snr, exceed_lo=np.sum(diff > tie, axis=1), exceed_hi=np.sum(diff >= -tie, axis=1))


def fp_statistic(Ct, seg_off, seg_len, rows, dot2=None):
    """Reference of ptar_fp_project + ptar_fp_reduce.  ``Ct`` [n, 2 Nf] per pulsar (engine.fp_whitened_basis) as a
    list; returns amps [R, P, 2 Nf] and Fp [R, Nf] (check dicts)."""
    R, P = rows.shape[0], len(seg_off)
    nc = Ct[0].shape[1]
    h, l, b, t = (np.zeros((R, P, nc)) for _ in range(4))
    for a in range(P):
        Z = np.zeros((rows.shape[1], nc))
        Z[seg_off[a]:seg_off[a] + seg_len[a]] = Ct[a]
        h[:, a], l[:, a], b[:, a], t[:, a] = projection(rows, Z, seg_off[a], seg_len[a], dot2)
    Nf = nc // 2
    ah = h.reshape(R, P, Nf, 2).transpose(0, 2, 1, 3).reshape(R, Nf, 2 * P)
    al = l.reshape(R, P, Nf, 2).transpose(0, 2, 1, 3).reshape(R, Nf, 2 * P)
    ab = b.reshape(R, P, Nf, 2).transpose(0, 2, 1, 3).reshape(R, Nf, 2 * P)
    fh, fl = xsum_prod(ah, al, ah, al, dot2=dot2)
    fh, fl = 0.5 * fh, 0.5 * fl
    fb = np.sum(np.abs(ah) * ab, axis=-1) + gamma(2 * P + 8) * fh
    tt = t.reshape(R, P, Nf, 2).transpose(0, 2, 1, 3).reshape(R, Nf, 2 * P)
    return dict(amps=_out(h, l, b, t), Fp=_out(fh, fl, fb, 0.5 * np.sum(tt * tt, axis=-1)))


def timing_fit(T, rows, dot2=None):
    """Reference of ptar_timing_project on ``rows`` [R, ld]: post-fit rows (check dict over the TOAs of pulsars with a
    model; every other entry must be untouched).  ``T``: dict k [P], q_off, Q (flat, [k][n] per pulsar), sqrtw [ld],
    seg_off, seg_len."""
    h, l = rows.copy(), np.zeros_like(rows)
    b, t = np.zeros_like(rows), np.abs(rows)
    for a in range(len(T["k"])):
        k, s, n = int(T["k"][a]), int(T["seg_off"][a]), int(T["seg_len"][a])
        if k == 0:
            continue
        Q = T["Q"][T["q_off"][a]:T["q_off"][a] + k * n].reshape(k, n).T                   # [n, k]
        sw, r = T["sqrtw"][s:s + n], rows[:, s:s + n]
        yh, yl = two_prod(r, sw)
        ch, cl = xmatmul(yh, Q, dot2)
        ch, cl = fast_two_sum(ch, cl + yl @ Q)
        cb = gamma(n + 9) * (np.abs(yh) @ np.abs(Q))
        dh, dl = xmatmul(ch, Q.T, dot2)
        dh, dl = fast_two_sum(dh, dl + cl @ Q.T)
        db = cb @ np.abs(Q.T) + gamma(k) * (np.abs(ch) @ np.abs(Q.T))
        dt = (np.abs(yh) @ np.abs(Q)) @ np.abs(Q.T)
        eh, el = xdiv(dh, dl, sw)
        eb = db / sw + gamma(2) * np.abs(eh)
        ph, pl = xsub(r, eh, el)
        h[:, s:s + n], l[:, s:s + n] = ph, pl
        b[:, s:s + n] = eb + U * np.abs(ph)
        t[:, s:s + n] = np.abs(r) + dt / sw
    return _out(h, l, b, t)


# ------------------------------------------------------------------ Q(P, x), integer P
_HALF_LN_2PI = "0.91893853320467274178032973640561764"   # 1/2 ln(2 pi), parsed at the precision of the dtype


def q_int(P, x, dtype=np.float64):
    """Q(P, x) = Gamma(P, x) / Gamma(P) = e^-x sum_{k < P} x^k / k! for an integer P >= 1, vectorised over x >= 0:
    the largest term t_m (m = min(P - 1, floor x)) in log space -- m log1p((x - m) / m) + (m - x) - 1/2 ln(2 pi m) -
    delta(m), delta the Stirling series (m >= 16) or ln m! of the exact m! -- then the others by the ratios k / x (down)
    and x / (k + 1) (up), all <= 1.  ``dtype`` np.float64 restates the device's fp_q_int; np.longdouble is the
    reference."""
    x = np.atleast_1d(np.asarray(x, dtype=dtype))
    one = dtype(1)
    m = np.where(x < P - 1, np.floor(x), P - 1).astype(np.int64)
    dm = m.astype(dtype)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        fact = np.cumprod(np.r_[one, np.arange(1, 16, dtype=dtype)])                     # k! for k < 16, exact
        small = dm * np.log(x) - x - np.log(fact[np.minimum(m, 15)])
        i1 = one / np.maximum(dm, one)
        i2 = i1 * i1
        delta = i1 * (one / 12 - i2 * (one / 360 - i2 * (one / 1260 - i2 * (one / 1680 - i2 * (one / 1188)))))
        big = dm * np.log1p((x - dm) / np.maximum(dm, one)) + (dm - x) - (dtype(_HALF_LN_2PI) + np.log(np.maximum(dm, one)) / 2) - delta
        L = np.where(m == 0, -x, np.where(m < 16, small, big))
        s, r = np.ones_like(x), np.ones_like(x)
        for k in range(int(m.max()), 0, -1):
            live = k <= m
            r = np.where(live, r * (dtype(k) / x), r)
            s = np.where(live, s + r, s)
        r = np.ones_like(x)
        for k in range(int(m.min()) + 1, P):
            live = k > m
            r = np.where(live, r * (x / dtype(k)), r)
            s = np.where(live, s + r, s)
        q = np.exp(L) * s
    return np.where(x == 0, one, np.where(np.isinf(x), dtype(0), q))


# ------------------------------------------------------------------ edge batches
def edge_pulsars(ntoas, seed=0, span=(53000.0, 58800.0), name="E"):
    """Synthetic pulsars with the given TOA counts: epochs of 1-4 sub-band TOAs within 1 s spread over ``span`` (MJD),
    backends A/B/C cycling per epoch (flag f), uncertainties 0.3-3 us, isotropic sky positions."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, n in enumerate(ntoas):
        sub = []
        while sum(sub) < n:
            sub.append(int(min(rng.integers(1, 5), n - sum(sub))))
        ep = np.sort(rng.uniform(span[0], span[1], len(sub)))
        mjd = np.concatenate([e + np.sort(rng.uniform(0, 0.9, k)) / 86400.0 for e, k in zip(ep, sub)])
        be = np.concatenate([[("A", "B", "C")[q % 3]] * k for q, k in enumerate(sub)])
        ra, dec = rng.uniform(0, 24), math.degrees(math.asin(rng.uniform(-1, 1)))
        p = pulsar_from_arrays(f"{name}{j:03d}", {"RAJ": float(ra), "DECJ": float(dec)}, mjd.astype(np.longdouble),
                               rng.uniform(0.3, 3.0, n), flags=[{"f": f} for f in be])
        make_ideal(p)
        out.append(p)
    return out


def edge_batch(ntoas, seed=0, tm_min=16, plan_only=False, red=True, ecorr=True, tm=True):
    """A PulsarBatch of ``edge_pulsars`` with white + ECORR + red noise and, on pulsars of >= ``tm_min`` TOAs, a
    ``poly=2, jumps="f"`` timing model."""
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(edge_pulsars(ntoas, seed), plan_only=plan_only)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.1, log10_equad=-6.5)
        if ecorr:
            b.set_ecorr(i, -6.3, coarsegrain=1.0 / 86400.0)
        if red:
            b.set_red(i, -13.8 - 0.01 * (i % 10), 3.5 + 0.03 * (i % 10), components=10)
        if tm and b.ntoa[i] >= tm_min:
            b.set_timing_model(i, poly=2, jumps="f")
    return b


# TOA counts at the kernel edges: the only chunk partial (5, 6, 7), one chunk exactly (64), one TOA past it (65),
# 4 chunks of 64 with a partial last one so the 3-stage ring wraps (193), tile splits at 1024 (1025, 2100: 3 tiles)
EDGE_NTOAS = (5, 6, 7, 64, 65, 193, 1025, 2100)
OS_K = (1, 4, 5, 8, 9, 12, 13, 16)              # ncp = 8, 8, 16, 16, 24, 24, 32, 32
FP_NF = (1, 31, 32, 33, 100, 255, 256)          # n_cb = 1, 1, 1, 2, 4, 8, 8
TM_KMAX = (1, 4, 5, 8, 9, 16, 17, 32)           # column buckets 4, 4, 8, 8, 16, 16, 32, 32


def tm_columns(b, i, k):
    """``k`` timing-model columns for pulsar ``i``: poly (degree <= 2) plus smooth sinusoids of the span ('extra',
    table order), as set_timing_model(i, poly=..., extra=...) arguments."""
    poly = min(k, 3) - 1
    m = k - (poly + 1)
    t = np.asarray(b.psrs[i].toas.table["tdbld"], dtype=float) * 86400.0
    x = (t - t.min()) / (t.max() - t.min())
    ex = [np.sin(np.pi * (q // 2 + 1) * x + (q % 2) * np.pi / 2) for q in range(m)]
    return poly, (np.stack(ex, axis=1) if m else None)


def os_cases():
    """(K, templates, R) of the optimal-statistic sweep: every K, one or four templates (the 4th a random symmetric
    matrix), R across the realization-block edges."""
    Rs = (1, 3, 63, 64, 65, 130, 1, 65)
    return [(K, "hd" if j % 2 == 0 else "all4", Rs[j]) for j, K in enumerate(OS_K)]


def fp_cases():
    """(Nf or 'unsorted', R) of the Fp sweep."""
    Rs = (1, 63, 64, 65, 130, 63, 65)
    return [(nf, Rs[j]) for j, nf in enumerate(FP_NF)] + [("unsorted", 130)]


def null_cases():
    """(method, n, K, n_psr, R) of the null sweep: one partial column block (n + 1 < 64), exactly one (64), one column
    past it (65), several (201); kd < 32 (P = 2, K = 1..5 phase shifts); P = 2, 3, 24."""
    return [("phase_shift", 1, 1, 2, 1), ("phase_shift", 63, 5, 2, 65), ("phase_shift", 64, 16, 3, 130),
            ("phase_shift", 200, 5, 24, 65), ("sky_scramble", 63, 1, 3, 130), ("sky_scramble", 64, 16, 24, 65),
            ("sky_scramble", 200, 5, 3, 1), ("phase_shift", 63, 16, 24, 1)]


def random_template(P, seed=0):
    rng = np.random.default_rng(seed)
    G = rng.uniform(-0.5, 0.5, (P, P))
    return 0.5 * (G + G.T)


def templates(P, kind):
    return ("hd",) if kind == "hd" else ("hd", "monopole", "dipole", random_template(P))


def null_ntoas(P):
    return tuple(EDGE_NTOAS[(3 * j) % len(EDGE_NTOAS)] if P <= 3 else (5, 6, 7, 64, 65, 193)[j % 6] for j in range(P))
