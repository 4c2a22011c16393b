"""CPU tests of the extended-precision reference of the residual generator and the GWB stage
(tests/generator_reference.py): the reference is exact to well below its bounds, the bounds reject subtly wrong results
built in numpy, and the edge batches reach every kernel variant the GPU sweep claims."""
from fractions import Fraction

import numpy as np
import pytest

from tests import generator_reference as GR

U = GR.U
Fr = lambda x: Fraction(float(x))                               # noqa: E731


def _err(ref, idx, exact):
    return abs(Fr(ref["hi"][idx]) + Fr(ref["lo"][idx]) - exact) / Fraction(float(ref["bound"][idx]))


# ------------------------------------------------------------------ a small synthetic case of every stage
def _case(seed=0, R=6, gwb=True, conv=False):
    """Statics of a plan_only edge batch with random O(1) basis, coefficients, grid and weights (dt of up to ~1 s and
    omega ~ 1, so that every term of the Taylor step is far above the rounding of the others)."""
    rng = np.random.default_rng(seed)
    b = GR.gen_batch(ntoas=(1, 5, 17, 70, (16, 1), (17, 2), (33, 4)), dense=(3,), seed=seed, plan_only=True, red=3,
                     det=True, two_draws=True, conv=conv,
                     gwb=dict(log10_amplitude=-14.5, spectral_index=13 / 3, npts=30, howml=1) if gwb else None,
                     rn_taylor_tol=1e-18)                                        # nd = 3 wherever an epoch has a span
    pl = b.plan()
    J, P = pl["J"], b.n_psr
    S = {k: pl[k] for k in ("w1", "w2", "dtau", "det", "ep_gidx", "ep_gw", "ep_ecorr", "ep_bucket", "psr_bucket_off")}
    S.update(tiles=pl["tiles"], J=J, ld=b.ld, flags=pl["flags"], conv=int(conv), eloc=pl["eloc"])
    S["ep_ginv"] = pl["ep_ginv"] * 1e6                            # slopes of O(1) per second
    S["Ftile"] = rng.standard_normal(len(pl["tiles"]) * J * GR.EP)
    S["rn_scale"] = rng.uniform(0.5, 2.0, (P, J))
    S["rn_omega"] = rng.uniform(0.5, 2.0, (P, J // 2))
    S["G"] = rng.standard_normal((pl["g_ld"], R)) if gwb else None
    D = dict(z1=rng.standard_normal((R, b.ld)), z2=rng.standard_normal((R, b.ld)),
             zb=rng.standard_normal((R, pl["n_bucket_total"])), zrn=rng.standard_normal((R, P, J)))
    return b, pl, S, D


def _exact_toa(S, D, r, gi, tile):
    """y of one (realization, TOA) in exact rational arithmetic."""
    ts, n, loc0, ep0, nep, psr, nd, _ = tile
    J = S["J"]
    e = int(S["eloc"][gi])
    ge = ep0 + e
    sgn = Fraction(1 if S["conv"] else -1)
    F = S["Ftile"][S["tiles"].tolist().index(list(tile)) * J * GR.EP:][:J * GR.EP].reshape(J, GR.EP)[:, e]
    s, w, z = S["rn_scale"][psr], S["rn_omega"][psr], D["zrn"][r, psr]
    c = [Fraction(0)] * 3
    for j in range(J):
        a = Fr(s[j]) * Fr(z[j])
        k, odd = j // 2, j % 2
        pa = Fr(s[j + 1 - 2 * odd]) * Fr(z[j + 1 - 2 * odd])
        A = (a, (sgn if not odd else -sgn) * Fr(w[k]) * pa, -Fraction(1, 2) * Fr(w[k]) ** 2 * a)
        for d in range(nd):
            c[d] += Fr(F[j]) * A[d]
    if S["G"] is not None:
        g0, g1 = Fr(S["G"][S["ep_gidx"][ge], r]), Fr(S["G"][S["ep_gidx"][ge] + 1, r])
        c[0] += g0 + Fr(S["ep_gw"][ge]) * (g1 - g0)
        c[1] += (g1 - g0) * Fr(S["ep_ginv"][ge])
    c[0] += Fr(S["ep_ecorr"][ge]) * Fr(D["zb"][r, S["psr_bucket_off"][psr] + S["ep_bucket"][ge]])
    dt = Fr(S["dtau"][gi]) if nd > 1 else Fraction(0)
    y = sum((c[d] * dt ** d for d in range(nd)), Fraction(0))
    return y + Fr(S["det"][gi]) + Fr(S["w1"][gi]) * Fr(D["z1"][r, gi]) + Fr(S["w2"][gi]) * Fr(D["z2"][r, gi])


def test_reference_is_exact_to_well_below_its_bounds():
    """Every stage against Fraction sums on small random cases: error <= 1e-3 of the bound."""
    b, pl, S, D = _case(R=3)
    R = 3
    ref, _ = GR.generate(S, D, R)
    rng = np.random.default_rng(1)
    worst = Fraction(0)
    tiles = [tuple(t) for t in pl["tiles"].tolist()]
    for tile in tiles[:: max(1, len(tiles) // 8)] + tiles[-2:]:
        for gi in rng.choice(np.arange(tile[0], tile[0] + tile[1]), min(tile[1], 3), replace=False):
            for r in range(R):
                worst = max(worst, _err(ref, (r, gi), _exact_toa(S, D, r, int(gi), tile)))
    P, Jg = b.n_psr, 12
    z = rng.standard_normal((R, P, Jg))
    M = np.tril(rng.standard_normal((P, P)))
    mix = GR.mix(M, z)
    for p, r, j in zip(rng.integers(0, P, 20), rng.integers(0, R, 20), rng.integers(0, Jg, 20)):
        ex = sum((Fr(M[p, q]) * Fr(z[r, q, j]) for q in range(p + 1)), Fraction(0))
        worst = max(worst, _err(mix, (p, r, j), ex))
    A = rng.standard_normal((30, Jg)) * np.exp(rng.uniform(-5, 5, (30, Jg)))
    Zm = mix["hi"]
    syn = GR.synth(A, Zm, pl["knots"], pl["syn_tiles"])
    cols = GR._columns(pl["knots"], pl["syn_tiles"])
    for c in np.flatnonzero(cols >= 0)[::7]:
        for r in range(R):
            ex = sum((Fr(A[pl["knots"][c], j]) * Fr(Zm[cols[c], r, j]) for j in range(Jg)), Fraction(0))
            worst = max(worst, _err(syn, (c, r), ex))
    print(f"\n[generator reference] worst error / bound {float(worst):.1e}")
    assert worst <= Fraction(1, 1000)


def test_int8_reference_is_the_exact_integer_product():
    """synth_i8 against the digit product formed with Python integers: error <= 1e-3 of the bound; the full six-digit
    product (keep = 11 diagonals) is within 2^-44 of the unquantised one relative to full scale."""
    rng = np.random.default_rng(3)
    R, P, J = 5, 2, 40
    A = np.tril(rng.standard_normal((12, J)))
    sA = 2.0 ** (np.ceil(np.log2(np.abs(A).max(axis=1))) + 2)
    Zm = rng.standard_normal((P, R, J))
    zs = 2.0 ** (np.ceil(np.log2(np.abs(Zm).reshape(P, -1).max(axis=1))) + 2)
    knots = np.r_[np.arange(0, 7), -1, np.arange(3, 12)].astype(np.int32)
    tiles = np.array([[0, 0, 7, 7], [1, 8, 9, 12]], dtype=np.int32)
    ref = GR.synth_i8(A, sA, Zm, zs, knots, tiles)
    assert np.all(ref["hi"][7] == 0) and np.all(ref["bound"][7] == 0)
    worst = Fraction(0)
    cols = GR._columns(knots, tiles)
    for c in np.flatnonzero(cols >= 0):
        p, k = cols[c], knots[c]
        ad = GR.digits(A[k] / sA[k]).astype(np.int64)
        for r in range(R):
            zd = GR.digits(Zm[p, r] / zs[p]).astype(np.int64)
            E = sum(Fraction(int(np.dot(zd[s], ad[t])), 256 ** (s + t)) for s in range(6) for t in range(6) if s + t <= 6)
            ex = E * Fr(sA[k]) * Fr(zs[p]) / 2 ** 16
            worst = max(worst, _err(ref, (c, r), ex))
    assert worst <= Fraction(1, 1000)
    full = GR.synth_i8(A, sA, Zm, zs, knots, tiles, keep=11)
    m = cols >= 0
    assert np.max(np.abs(full["hi"][m] - full["exact"][m])) <= 2.0 ** -44 * np.max(np.abs(full["exact"]))


# ------------------------------------------------------------------ mutations
def _emulate(S, D, R, mut=()):
    """The generator in plain fp64, the kernel's operation order, with optional mutations."""
    J, ld = S["J"], S["ld"]
    out = np.zeros((R, ld))
    tiles = S["tiles"]
    for ti, (ts, n, loc0, ep0, nep, psr, nd, _) in enumerate(tiles.tolist()):
        s, w, z = S["rn_scale"][psr], S["rn_omega"][psr], D["zrn"][:R, psr]
        sgn = (1.0 if S["conv"] else -1.0) * (-1.0 if ("A1 sign" in mut and psr == 1) else 1.0)
        a = s * z
        A1 = np.empty_like(a)
        A1[:, 0::2], A1[:, 1::2] = sgn * w * a[:, 1::2], -sgn * w * a[:, 0::2]
        h = (-1.0 if "A2 half" in mut else -0.5) * w * w
        A2 = np.repeat(h, 2) * a
        F = S["Ftile"][ti * J * GR.EP:(ti + 1) * J * GR.EP].reshape(J, GR.EP)[:, :nep]
        c = [x @ F if d < nd else np.zeros((R, nep)) for d, x in enumerate((a, A1, A2))]
        if "split-K twice" in mut and nep <= 16:
            c = [x + (y[:, J // 4:J // 2] @ F[J // 4:J // 2] if d < nd else 0) for d, (x, y) in enumerate(zip(c, (a, A1, A2)))]
        ge = np.arange(ep0, ep0 + nep)
        G = S["G"]
        g0, g1 = G[S["ep_gidx"][ge], :R].T, G[S["ep_gidx"][ge] + 1, :R].T
        dg = g1 - g0
        add0, add1 = S["ep_gw"][ge] * dg + g0, dg * S["ep_ginv"][ge]
        if "slope on c0" in mut:
            add0, add1 = add0 + add1, 0.0 * add1
        bk = S["ep_bucket"][ge] + (1 if "ECORR b+1" in mut else 0)
        bk = np.minimum(bk, np.r_[S["psr_bucket_off"][1:], D["zb"].shape[1]][psr] - 1 - S["psr_bucket_off"][psr]) \
            if "ECORR b+1" in mut else bk
        add0 = add0 + S["ep_ecorr"][ge] * D["zb"][:R, S["psr_bucket_off"][psr] + bk]
        c[0], c[1] = c[0] + add0, c[1] + add1
        gi = np.arange(ts, ts + n)
        el = S["eloc"][gi].astype(np.int64)
        if "eloc+1" in mut and nep > 1:
            el = np.where(el == 0, 1, el)
        dt = S["dtau"][gi] if nd > 1 else 0.0 * gi
        v = c[0][:, el] + dt * (c[1][:, el] + dt * c[2][:, el]) if nd > 2 else c[0][:, el] + dt * c[1][:, el]
        v = v + S["det"][gi] + S["w1"][gi] * D["z1"][:R, gi] + S["w2"][gi] * D["z2"][:R, gi]
        if "drop last TOA" in mut and n % 4 == 1:
            v[:, -1] = 0.0
        out[:, gi] = v
    return out


def test_generator_mutations_are_rejected():
    b, pl, S, D = _case(R=5)
    R = 5
    ref, written = GR.generate(S, D, R)
    chk = lambda x, what: GR.check(x[:, written], {k: v[:, written] for k, v in ref.items()}, what)   # noqa: E731
    assert chk(_emulate(S, D, R), "fp64")[0] <= 1.0
    for mut in ("A1 sign", "A2 half", "slope on c0", "eloc+1", "drop last TOA", "split-K twice", "ECORR b+1"):
        with pytest.raises(AssertionError):
            chk(_emulate(S, D, R, (mut,)), mut)


def test_gwb_mutations_are_rejected():
    """Mix with one M[p][q] above the diagonal; synthesis with a pad knot gathering row 0 and with the k-range cut at
    kend - 1; int8 synthesis with the diagonal d = 6 dropped."""
    rng = np.random.default_rng(4)
    R, P, J = 7, 5, 24
    z = rng.standard_normal((R, P, J))
    M = np.tril(rng.standard_normal((P, P)))
    good = np.einsum("pq,rqj->prj", M, z)
    assert GR.check(good, GR.mix(M, z), "mix")[0] <= 1.0
    Mu = M.copy()
    Mu[1, 3] = 0.3
    with pytest.raises(AssertionError):
        GR.check(np.einsum("pq,rqj->prj", Mu, z), GR.mix(Mu, z), "M above the diagonal")
    A = np.tril(rng.standard_normal((J, J)))
    knots = np.r_[0, 3, 9, -1, 2, 5, 11, 17].astype(np.int32)
    tiles = np.array([[0, 0, 3, 10], [1, 4, 4, 18]], dtype=np.int32)
    cols = GR._columns(knots, tiles)
    ref = GR.synth(A, good, knots, tiles)

    def G_of(kcut=None, pad_row0=False):
        G = np.zeros((len(knots), R))
        for c in range(len(knots)):
            if cols[c] >= 0:
                kend = tiles[cols[c], 3] if kcut is None else kcut[cols[c]]
                G[c] = good[cols[c], :, :kend] @ A[knots[c], :kend]
            elif pad_row0:
                G[c] = good[0] @ A[0]
        return G
    assert GR.check(G_of(), ref, "synth")[0] <= 1.0
    for what, G in (("pad knot gathers row 0", G_of(pad_row0=True)), ("kend - 1", G_of(kcut=tiles[:, 3] - 1))):
        with pytest.raises(AssertionError):
            GR.check(G, ref, what)
    sA = 2.0 ** (np.ceil(np.log2(np.abs(A).max(axis=1))) + 2)
    zs = 2.0 ** (np.ceil(np.log2(np.abs(good).reshape(P, -1).max(axis=1))) + 2)
    ri8 = GR.synth_i8(A, sA, good, zs, knots, tiles)
    assert GR.check(ri8["hi"], ri8, "i8")[0] <= 1.0
    with pytest.raises(AssertionError):
        GR.check(GR.synth_i8(A, sA, good, zs, knots, tiles, keep=6)["hi"], ri8, "d = 6 dropped")


# ------------------------------------------------------------------ coverage
def test_edge_batches_reach_every_claimed_variant():
    """The GPU sweep's batches (plan_only): tiles in every split-K class and at exactly 16, 17, 32, 33, 64 epochs; nd 1,
    2, 3 mixed inside one tile; n_toa of 1 ... 1024 with every residue mod 4; an epoch split across two tiles; full
    64-knot blocks, partial ones down to 2 knots and odd counts (a pad knot); kend % 16 != 0; the first and last grid
    interval."""
    from pta_replicator_b200 import _cabi
    gw = dict(log10_amplitude=-14.5, spectral_index=13 / 3, npts=150, howml=3)
    seen = dict(n_ep=set(), res=set(), nd_mixed=False, split_epoch=False, knots=set(), odd=False, kend16=False,
                first=False, last=False, ntoa=set())
    for kw in (dict(gwb=gw), dict(conv=True, red=31, rn_taylor_tol=1e-14, gwb=dict(gw, npts=20, howml=1))):
        b = GR.gen_batch(plan_only=True, **kw)
        pl = b.plan()
        t = pl["tiles"]
        seen["n_ep"] |= set(t[:, 4].tolist())
        seen["ntoa"] |= set(t[:, 1].tolist())
        seen["res"] |= set((t[:, 1] % 4).tolist())
        for i in range(b.n_psr):
            ep, first, nd, _, gj = b._epochs_for(i, 0.0)
            for ts, n, loc0, ep0, nep in t[t[:, 5] == i][:, :5].tolist():
                e0 = ep0 - int(np.sum([len(b._epochs_for(k, 0.0)[1]) for k in range(i)]))
                nds = set(nd[e0:e0 + nep].tolist())
                seen["nd_mixed"] |= len(nds) >= 2 and 3 in nds
            loc = t[t[:, 5] == i]
            for a, c in zip(loc[:-1], loc[1:]):
                seen["split_epoch"] |= int(ep[a[2] + a[1] - 1]) == int(ep[c[2]])
            seen["first"] |= int(gj.min()) == 0
            seen["last"] |= int(gj.max()) == pl["knots"].max() - 1 or int(gj.max()) == kw["gwb"]["npts"] - 2
        st = pl["syn_tiles"]
        seen["knots"] |= set(st[:, 2].tolist())
        seen["odd"] |= bool(np.any(pl["knots"] < 0))
        seen["kend16"] |= bool(np.any(st[:, 3] % 16 != 0))
    print(f"\n[coverage] n_ep {sorted(seen['n_ep'])}\n  n_toa {sorted(seen['ntoa'])}\n  knot blocks {sorted(seen['knots'])}")
    assert {16, 17, 32, 33, 64} <= seen["n_ep"]
    assert min(seen["n_ep"]) <= 16 and any(16 < n <= 32 for n in seen["n_ep"]) and any(n > 32 for n in seen["n_ep"])
    assert seen["res"] == {0, 1, 2, 3} and {1, 2, 3} <= seen["ntoa"] and max(seen["ntoa"]) == _cabi.TILE_TOAS
    assert seen["nd_mixed"] and seen["split_epoch"]
    assert 64 in seen["knots"] and min(seen["knots"]) <= 2 and any(k % 2 for k in seen["knots"])
    assert seen["odd"] and seen["kend16"] and seen["first"] and seen["last"]
