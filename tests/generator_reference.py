"""Extended-precision reference of the residual generator and the GWB stage -- ``ptar_gwb_mix``, ``ptar_gwb_synth`` (fp64
DMMA), ``ptar_gwb_synth_i8`` (int8 digit slices) and ``ptar_generate`` (fused, two-kernel and rc = 32 schedules) -- with a
rigorous componentwise error bound per output; numpy only, no torch.

The reference evaluates the operation the kernels evaluate on the fp64 statics the device holds (pulled back from
``compile()``: tiles, Ftile, rn_scale, rn_omega, dtau, eloc, ep_*, w1 / w2 / wm, det, M, gwb_T / gwb_L, knots, syn_tiles,
i8_*), so only kernel arithmetic is under test; the physics is the oracle tests' business.  Values are unevaluated pairs
hi + lo; the pair arithmetic, ``Report`` and ``check`` are those of tests/reduction_reference.py.  Draws are either
injected or the device's own normal stream (``ptar_philox_normals`` evaluates the same ``normals4`` as the kernels; the
GPU tests prove the bit-identity before they rely on it).

Operations and bounds (u = 2^-53, gamma_m = m u / (1 - m u); every bound holds for any summation order, tensor-core
fragment order, k-split or split-K reduction, because it is a sum over |terms| with one gamma for the whole sum):

* Mix: Zm[p][r][j] = sum_{q <= p} M[p][q] z[r][q][j].  |d| <= gamma_{P+8} sum_q |M[p][q] z[r][q][j]|.
* DMMA synthesis: G[col][r] = sum_{j < J} A[knot(col)][j] Zm[p][r][j] over the compact knot columns of pulsar p.
  |d| <= gamma_{J+8} sum_j |A Zm|.  The sum runs over all J columns: a lower-triangular A is zero past its diagonal, so
  the kernel's cut at ``kend`` is exact, and a cut one column short is an error.  Pad columns (knot -1) must be exactly 0.
* int8 synthesis: the kernel multiplies the digits a_t = radix256_digits(A / sA) and z_s of round(Zm 2^48 / zscale[p])
  exactly in int32 and keeps the diagonals d = s + t <= 6: E = sum_{d <= 6} 2^(-8 d) D_d, D_d = sum_{s + t = d} z_s . a_t,
  G = E colscale zscale (powers of two: exact).  The reference forms the D_d exactly (integer-valued fp64 products whose
  partial sums stay below 2^53) and E as a pair; the device folds the seven diagonals with fp64 FMAs:
  |d| <= gamma_7 sum_d 2^(-8 d) |D_d| colscale zscale.  The distance to the unquantised product sum_j A Zm is reported for
  information only.
* Generator, per (tile epoch e, realization r), following ``rn_coefficients`` exactly:
    A_0 = s z,  A_1[2k] = +/-w_k s_{2k+1} z_{2k+1},  A_1[2k+1] = -/+w_k s_{2k} z_{2k} (+ for rn_convention = 1),
    A_2 = -1/2 w_k^2 s z,                                                       (s = rn_scale, w = rn_omega)
    c_d = sum_j F[j][e] A_d[j] (d < nd of the tile),
    c_0 += g0 + gw (g1 - g0) + ecorr z_b,   c_1 += (g1 - g0) ginv              (GWB grid, ECORR draw of the bucket)
  and per TOA  y = c_0 + dt c_1 + dt^2 c_2 (nd terms, dt = dtau) + det + w1 z1 (+ w2 z2).
  The A_d carry up to three roundings each (s z, the w factor, w^2) and the GEMM J terms, so
    |d c_d| <= gamma_{J+16} S_d,  S_0 = sum_j |F A_0| + |g0| + |gw| (|g0| + |g1|) + |ecorr z_b|,
                                  S_1 = sum_j |F A_1| + |ginv| (|g0| + |g1|),  S_2 = sum_j |F A_2|
  (the addends take at most four roundings: g1 - g0, the fma, ecorr z_b and the two adds).  Through Horner, to first
  order:  |d y| <= B_0 + |dt| B_1 + dt^2 B_2 + gamma_6 (|c_0| + B_0 + |dt| (|c_1| + B_1) + dt^2 (|c_2| + B_2) + |det|
  + |w1 z1| + |w2 z2|)  -- two Horner FMAs, the det add and two white FMAs.  Alignment slots after a pulsar's last TOA
  are exactly 0.

The last part builds the edge batches the CPU and GPU tests share."""
from __future__ import annotations

import math

import numpy as np

from tests.reduction_reference import (U, Report, check, fast_two_sum, gamma, two_prod, two_sum,  # noqa: F401
                                       xmatmul, xscale)

F_WHITE, F_ECORR, F_RED, F_GWB, F_DET, F_WHITE1 = 1, 2, 4, 8, 16, 32
EP = 64                                            # kernel-epochs per tile


def _out(h, l, bound, terms):
    return dict(hi=h, lo=l, bound=bound, terms=terms)


def pair_add(ah, al, bh, bl):
    s, e = two_sum(ah, bh)
    return fast_two_sum(s, e + (al + bl))


def pair_mul(ah, al, bh, bl):
    p, e = two_prod(ah, bh)
    return fast_two_sum(p, e + (ah * bl + al * bh))


def _pmatmul(h, l, B):
    """(h + l) @ B, B fp64: pair."""
    ph, pl = xmatmul(h, B)
    return fast_two_sum(ph, pl + l @ B)


# ------------------------------------------------------------------ GWB stage
def mix(M, z):
    """Zm [P, R, J] = tril(M) applied to z [R, P, J] over the pulsar axis (check dict)."""
    R, P, J = z.shape
    Mt = np.tril(np.asarray(M, dtype=np.float64).reshape(P, P))
    Z = np.ascontiguousarray(z.transpose(0, 2, 1)).reshape(R * J, P)
    h, l = xmatmul(Z, Mt.T)
    t = np.abs(Z) @ np.abs(Mt.T)
    f = lambda a: a.reshape(R, J, P).transpose(2, 0, 1)       # noqa: E731
    return _out(f(h), f(l), gamma(P + 8) * f(t), f(t))


def _columns(knots, syn_tiles):
    """Pulsar of every compact grid column (-1: pad column) from the tile list (pulsar, first column, count, kend)."""
    psr = np.full(len(knots), -1, dtype=np.int64)
    for p, kn0, cnt, _ in np.asarray(syn_tiles).reshape(-1, 4).tolist():
        psr[kn0:kn0 + cnt] = p
    return psr


def synth(A, Zm, knots, syn_tiles):
    """G [g_ld, R] = sum_j A[knot][j] Zm[p][r][j] per compact column; pad columns exactly 0 (check dict).  ``A`` [npts, J]
    (J = the leading dimension the device uses), ``Zm`` [P, R, J]."""
    P, R, J = Zm.shape
    knots = np.asarray(knots)
    psr = _columns(knots, syn_tiles)
    h, l, t = (np.zeros((len(knots), R)) for _ in range(3))
    for p in range(P):
        cols = np.flatnonzero(psr == p)
        if cols.size == 0:
            continue
        Ak = A[knots[cols], :J]
        gh, gl = xmatmul(Zm[p], Ak.T)
        h[cols], l[cols], t[cols] = gh.T, gl.T, (np.abs(Zm[p]) @ np.abs(Ak.T)).T
    return _out(h, l, gamma(J + 8) * t, t)


def digits(x, nslices=6):
    """Signed radix-256 digits (PulsarBatch.radix256_digits) as fp64: [nslices, ...]."""
    from pta_replicator_b200.engine import PulsarBatch
    return PulsarBatch.radix256_digits(x, nslices).astype(np.float64)


def synth_i8(A, sA, Zm, zscale, knots, syn_tiles, keep=7):
    """Reference of ptar_gwb_synth_i8 on the operands as the kernel sees them (check dict [g_ld, R] plus ``exact``, the
    unquantised product, for information).  ``sA`` per row of A, ``zscale`` per pulsar; ``keep`` diagonals."""
    P, R, J = Zm.shape
    knots = np.asarray(knots)
    psr = _columns(knots, syn_tiles)
    h, l, b, t, xh = (np.zeros((len(knots), R)) for _ in range(5))
    for p in range(P):
        cols = np.flatnonzero(psr == p)
        if cols.size == 0:
            continue
        rows = knots[cols]
        ad = digits(A[rows, :J] / sA[rows, None])                   # [6, ncol, J]
        zd = digits(Zm[p] / zscale[p])                              # [6, R, J]
        eh, el, et = np.zeros((R, cols.size)), np.zeros((R, cols.size)), np.zeros((R, cols.size))
        for d in range(keep):
            Dd = sum(zd[s] @ ad[d - s].T for s in range(max(0, d - 5), min(d, 5) + 1))   # exact: |partial sums| < 2^53
            w = 2.0 ** (-8 * d)
            eh, el = pair_add(eh, el, Dd * w, 0.0)
            et += np.abs(Dd) * w
        sc = sA[rows] * 2.0 ** -16 * zscale[p]
        h[cols], l[cols] = (eh * sc).T, (el * sc).T
        b[cols], t[cols] = (gamma(7) * et * sc).T, (et * sc).T
        xh[cols] = (Zm[p] @ A[rows, :J].T).T
    out = _out(h, l, b, t)
    out["exact"] = xh
    return out


# ------------------------------------------------------------------ generator
def rn_coefficients(scale, omega, z, conv):
    """The three coefficient rows A_d [R, J] (pairs) of one pulsar: ``scale`` [J], ``omega`` [J/2], ``z`` [R, J]."""
    sgn = 1.0 if conv else -1.0
    a0 = two_prod(z, scale[None, :])
    we = np.repeat(omega, 2)[None, :]
    # A_1: column 2k takes +sgn w a_{2k+1}, column 2k+1 takes -sgn w a_{2k}
    sw = np.empty_like(z)
    sw[:, 0::2], sw[:, 1::2] = a0[0][:, 1::2], a0[0][:, 0::2]
    swl = np.empty_like(z)
    swl[:, 0::2], swl[:, 1::2] = a0[1][:, 1::2], a0[1][:, 0::2]
    f1 = np.broadcast_to(we * np.where(np.arange(z.shape[1]) % 2 == 0, sgn, -sgn)[None, :], z.shape)
    a1 = xscale(sw, swl, f1)
    w2h, w2l = two_prod(we, we)
    a2 = pair_mul(a0[0], a0[1], np.broadcast_to(-0.5 * w2h, z.shape), np.broadcast_to(-0.5 * w2l, z.shape))
    return a0, a1, a2


def generate(S, D, R):
    """Reference of ptar_generate: check dict over [R, ld] and the mask of the entries the kernel writes (TOAs and
    alignment slots).  ``S``: the statics (tiles [n, 8], J, conv, Ftile, rn_scale [P, J], rn_omega [P, J/2], w1, w2,
    dtau, eloc, det, ep_gidx, ep_gw, ep_ginv, ep_ecorr, ep_bucket, psr_bucket_off, flags (with F_WHITE1: one draw,
    w1 the merged weight), ld, G [g_ld, >= R] or None).  ``D``: draws z1, z2 [R, ld], zb [R, n_bucket_total],
    zrn [R, P, J] (absent terms may be None)."""
    ld, J, flags = S["ld"], S["J"], S["flags"]
    has_red = bool(flags & F_RED) and J > 0
    has_ecorr = bool(flags & F_ECORR)
    has_gwb = bool(flags & F_GWB) and S.get("G") is not None
    has_epoch = has_red or has_ecorr or has_gwb
    has_white = bool(flags & F_WHITE)
    two = has_white and not (flags & F_WHITE1)
    has_det = bool(flags & F_DET)
    h, l, b, t = (np.zeros((R, ld)) for _ in range(4))
    written = np.zeros(ld, dtype=bool)
    coef = {}
    for ti, (ts, n, loc0, ep0, nep, psr, nd, _) in enumerate(np.asarray(S["tiles"]).tolist()):
        gi = np.arange(ts, ts + n)
        written[ts:ts + ((n + 3) & ~3)] = True
        yh, yl = np.zeros((R, n)), np.zeros((R, n))
        mag = np.zeros((R, n))
        bnd = np.zeros((R, n))
        if has_epoch:
            c = [(np.zeros((R, nep)), np.zeros((R, nep))) for _ in range(3)]
            S_ = [np.zeros((R, nep)) for _ in range(3)]
            if has_red:
                if psr not in coef:
                    coef[psr] = rn_coefficients(S["rn_scale"][psr], S["rn_omega"][psr], D["zrn"][:R, psr, :], S["conv"])
                F = np.asarray(S["Ftile"][ti * J * EP:(ti + 1) * J * EP]).reshape(J, EP)[:, :nep]
                for d in range(min(nd, 3)):
                    ah, al = coef[psr][d]
                    c[d] = _pmatmul(ah, al, F)
                    S_[d] = np.abs(ah) @ np.abs(F)
            ge = np.arange(ep0, ep0 + nep)
            if has_gwb:
                G = S["G"]
                gidx = S["ep_gidx"][ge]
                g0, g1 = G[gidx, :R].T, G[gidx + 1, :R].T
                gw, ginv = S["ep_gw"][ge][None, :], S["ep_ginv"][ge][None, :]
                dgh, dgl = two_sum(g1, -g0)
                ph, pl = xscale(dgh, dgl, np.broadcast_to(gw, dgh.shape))
                c[0] = pair_add(*c[0], *pair_add(ph, pl, g0, 0.0))
                c[1] = pair_add(*c[1], *xscale(dgh, dgl, np.broadcast_to(ginv, dgh.shape)))
                S_[0] = S_[0] + np.abs(g0) + np.abs(gw) * (np.abs(g0) + np.abs(g1))
                S_[1] = S_[1] + np.abs(ginv) * (np.abs(g0) + np.abs(g1))
            if has_ecorr:
                zb = D["zb"][:R, S["psr_bucket_off"][psr] + S["ep_bucket"][ge]]
                eh, el = two_prod(zb, np.broadcast_to(S["ep_ecorr"][ge][None, :], zb.shape))
                c[0] = pair_add(*c[0], eh, el)
                S_[0] = S_[0] + np.abs(eh)
            B = [gamma(J + 16) * s for s in S_]
            el_ = S["eloc"][gi].astype(np.int64)
            dt = S["dtau"][gi][None, :] if nd > 1 else np.zeros((1, n))
            dtb = np.broadcast_to(dt, (R, n))
            yh, yl = c[0][0][:, el_], c[0][1][:, el_]
            bnd = B[0][:, el_].copy()
            mag = np.abs(yh) + B[0][:, el_]
            for d in range(1, min(nd, 3)):
                th, tl = c[d][0][:, el_], c[d][1][:, el_]
                for _ in range(d):
                    th, tl = xscale(th, tl, dtb)
                yh, yl = pair_add(yh, yl, th, tl)
                bnd += np.abs(dt) ** d * B[d][:, el_]
                mag += np.abs(th) + np.abs(dt) ** d * B[d][:, el_]
        if has_det:
            det = np.broadcast_to(S["det"][gi][None, :], (R, n))
            yh, yl = pair_add(yh, yl, det, 0.0)
            mag += np.abs(det)
        if has_white:
            ph, pl = two_prod(D["z1"][:R, gi], np.broadcast_to(S["w1"][gi][None, :], (R, n)))
            yh, yl = pair_add(yh, yl, ph, pl)
            mag += np.abs(ph)
            if two:
                ph, pl = two_prod(D["z2"][:R, gi], np.broadcast_to(S["w2"][gi][None, :], (R, n)))
                yh, yl = pair_add(yh, yl, ph, pl)
                mag += np.abs(ph)
        h[:, gi], l[:, gi] = yh, yl
        b[:, gi] = bnd + gamma(6) * mag
        t[:, gi] = mag
    return _out(h, l, b, t), written


# ------------------------------------------------------------------ edge batches
def dense_pulsars(ntoas, seed=0, span=(53000.0, 58800.0), name="D", dense=()):
    """Like reduction_reference.edge_pulsars (epochs of 1-4 sub-band TOAs within 1 s), but the pulsars listed in
    ``dense`` get epochs of 8-60 TOAs, so that an epoch straddles the 1024-TOA tile cut, and an entry (n_ep, k) of
    ``ntoas`` is a pulsar of exactly n_ep epochs of k TOAs."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, n in enumerate(ntoas):
        lo, hi = (8, 61) if j in dense else (1, 5)
        sub = []
        if isinstance(n, tuple):
            sub, n = [n[1]] * n[0], n[0] * n[1]
        while sum(sub) < n:
            sub.append(int(min(rng.integers(lo, hi), n - sum(sub))))
        ep = np.sort(rng.uniform(span[0], span[1], len(sub)))
        mjd = np.concatenate([e + np.sort(rng.uniform(0, 0.9, k)) / 86400.0 for e, k in zip(ep, sub)])
        be = np.concatenate([[("A", "B", "C")[q % 3]] * k for q, k in enumerate(sub)])
        ra, dec = rng.uniform(0, 24), math.degrees(math.asin(rng.uniform(-1, 1)))
        p = pulsar_from_arrays(f"{name}{j:03d}", {"RAJ": float(ra), "DECJ": float(dec)}, mjd.astype(np.longdouble),
                               rng.uniform(0.3, 3.0, n), flags=[{"f": f} for f in be])
        make_ideal(p)
        out.append(p)
    return out


# TOA counts at the generator's edges: 1-3 TOAs (a tile of one partial 4-group), every residue mod 4, 1023-1025 and
# ~2100 (tiles cut at 64 epochs); pulsar 9 is dense (8-60 TOAs per epoch: the 1024-TOA cut splits an epoch across two
# tiles); (n_ep, k) pulsars put tiles of exactly 16, 17, 32, 33 and 64 epochs at the split-K class edges (nsplit 4 for
# n_ep <= 16, 2 for <= 32, else 1)
GEN_NTOAS = (1, 2, 3, 5, 17, 1023, 1024, 1025, 2101, 2100, (16, 1), (17, 2), (32, 3), (33, 4), (64, 1))
GEN_DENSE = (9,)


def gen_batch(ntoas=GEN_NTOAS, dense=GEN_DENSE, seed=0, plan_only=False, white=True, two_draws=False, ecorr=True,
              red=10, gwb=None, det=False, conv=False, **kw):
    """A PulsarBatch of ``dense_pulsars`` with the chosen terms: ``red`` components (0: none), ``gwb`` a dict of set_gwb
    arguments (None: none), ``two_draws``: EQUAD as a second white draw, ``det``: a deterministic delay."""
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(dense_pulsars(ntoas, seed, dense=dense), plan_only=plan_only, **kw)
    T = float(np.ptp(np.concatenate(b.t_tdb)))                 # one frequency grid: a 1-TOA pulsar has no span of its own
    for i in range(b.n_psr):
        if white:
            b.set_white(i, efac=1.1, log10_equad=-6.5 if two_draws else None)
        if ecorr:
            b.set_ecorr(i, -6.3 - 0.05 * (i % 3), coarsegrain=1.0 / 86400.0)
        if red:
            with np.errstate(divide="ignore", invalid="ignore"):
                b.set_red(i, -13.8 - 0.01 * (i % 10), 3.5 + 0.03 * (i % 10), modes=np.arange(1, red + 1) / T,
                          libstempo_convention=conv)
        if red and not np.all(np.isfinite(b._red["scale"][i])):
            # a 1-TOA pulsar has no span: its prior 1/T is infinite; give it the prior of the longest pulsar
            b._red["scale"][i] = None
        if det:
            t = b.t_tdb[i]
            b.set_deterministic(i, (1e-7 * np.sin(2 * np.pi * (t - t[0]) / 3e7))[np.argsort(b.order[i])])
    if red:
        longest = int(np.argmax(b.ntoa))
        b._red["scale"] = [b._red["scale"][longest] if s is None else s for s in b._red["scale"]]
    if gwb is not None:
        b.set_gwb(**gwb)
    return b
