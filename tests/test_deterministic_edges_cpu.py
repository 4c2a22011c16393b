"""CPU tests of the extended-precision reference of the Fourier-basis, Cholesky, CW, CW-catalog, burst and memory
kernels (tests/deterministic_reference.py): the longdouble reference agrees with mpmath at 40 digits to well within its
bounds, the bounds reject subtly wrong results built in numpy, and the sweep's batches and catalogs reach the kernel
edges the GPU tests claim."""
import numpy as np
import pytest

from tests import deterministic_reference as DR

mp = DR.MK.mp


def _close_to_mp(E_val, mp_vals, what):
    """|longdouble - mpmath| <= 1e-3 bound at every point (``mp_vals`` a flat list of mpf)."""
    v, b = E_val.v.ravel(), E_val.e.ravel()
    worst = 0.0
    for k, x in enumerate(mp_vals):
        if mp.isnan(x):
            assert np.isnan(v[k]), (what, k)
            continue
        hi = float(v[k])
        d = float(abs(mp.mpf(hi) + mp.mpf(float(v[k] - DR.LD(hi))) - x)) if not np.isnan(v[k]) else np.inf
        assert d <= 1e-3 * b[k] or d == 0.0, f"{what} point {k}: |ld - mp| = {d:.3e}, bound {b[k]:.3e}"
        worst = max(worst, d / b[k] if b[k] else 0.0)
    return worst


def _mpf(x):
    return mp.mpf(float(x))


def _pre_points(n, seed):
    """fp64 prefactor rows of a random catalog, pulsar directions, and TOAs."""
    rng = np.random.default_rng(seed)
    cat = DR.catalog(n, seed=seed, merged=0.0)
    phat = DR.phat_of(rng.uniform(0, 2 * np.pi), np.arcsin(rng.uniform(-1, 1)))
    pre = DR.prefactors_np(cat, phat, 1.3, 0.0, 0)
    return cat, phat, pre


# ------------------------------------------------------------------ the reference against mpmath
def test_reference_against_mpmath_at_40_digits():
    mp.mp.dps = 40
    rng = np.random.default_rng(11)
    worst = {}
    # Fourier basis: arguments from ~1 to above 1e10 rad, with and without a phase
    n = 200
    t = rng.uniform(0, 5e9, n)
    f = 10.0 ** rng.uniform(-9.5, 0.5, n)
    ph = rng.uniform(0, 2 * np.pi, n)
    for phase in (None, ph):
        a = DR.fourier_arg(DR.EK, DR.E(t), DR.E(f), None if phase is None else DR.E(phase))
        assert np.abs(a.v).max() > 1e10 and np.abs(a.v).min() < 1e3
        for fn in ("sin", "cos"):
            ref = []
            for k in range(n):
                am = DR.fourier_arg(DR.MK, _mpf(t[k]), _mpf(f[k]), None if phase is None else _mpf(phase[k]))
                ref.append(getattr(DR.MK, fn)(am))
            worst["fourier"] = max(worst.get("fourier", 0), _close_to_mp(getattr(DR.EK, fn)(a), ref, f"fourier {fn}"))
    # catalog prefactors, both pulsar-distance branches
    cat, phat, _ = _pre_points(60, 12)
    for use_pphase in (0, 1):
        got = DR.prefactors(DR.EK, cat, phat, 1.3, 2.1, use_pphase)
        for k in range(cat.shape[1]):
            ref = DR.prefactors(DR.MK, cat[:, k], phat, 1.3, 2.1, use_pphase)
            for slot in range(14):
                g = DR.E(np.broadcast_to(got[slot].v, (cat.shape[1],))[k:k + 1],
                         np.broadcast_to(got[slot].e, (cat.shape[1],))[k:k + 1])
                worst["prefactors"] = max(worst.get("prefactors", 0), _close_to_mp(g, [ref[slot]], f"pre slot {slot}"))
    # CW evaluation, every mode x psr_term, including evolving points near merger
    _, _, pre = _pre_points(40, 13)
    t = rng.uniform(0, 5e8, 40)
    near = np.flatnonzero(pre[:, 1] * 5e8 > 1e-3)[:5]
    for k, s in enumerate(near):                                  # 1 - fac1 t from 1e-3 down to 1e-7
        t[s] = (1 - 10.0 ** -(3 + k)) / pre[s, 1]
    live = (1 - pre[:, 1] * t > 0) & (1 - pre[:, 1] * (t - pre[:, 13] * (1 - pre[:, 12])) > 0)
    pre, t = pre[live], t[live]
    assert (1 - pre[:, 1] * t).min() < 1e-6
    for mode in (0, 1, 2):
        for psr in (0, 1):
            got = DR.cw_res(DR.EK, DR.E(t), [DR.E(pre[:, j]) for j in range(14)], mode, psr)
            ref = [DR.cw_res(DR.MK, _mpf(t[k]), [_mpf(x) for x in pre[k, :14]], mode, psr) for k in range(len(t))]
            worst[f"cw mode {mode}"] = max(worst.get(f"cw mode {mode}", 0), _close_to_mp(got, ref, f"cw {mode} {psr}"))
    # Cholesky residual in pair arithmetic
    for n in (3, 17):
        A = DR.spd(n, 1e6, rng)
        L = np.linalg.cholesky(A)
        r = DR.cholesky_ref(A, L)
        for i in range(n):
            for j in range(i + 1):
                exact = mp.fsum(_mpf(L[i, k]) * _mpf(L[j, k]) for k in range(n))
                d = abs(_mpf(r["hi"][i, j]) + _mpf(r["lo"][i, j]) - exact)
                assert d <= 1e-3 * r["bound"][i, j] or d == 0
    print("\n[mpmath] worst |ld - mp| / bound: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items())))


def test_fp64_constants_are_the_kernels():
    from pta_replicator_b200 import constants as const
    assert (DR.SOLAR2S, DR.MPC2S, DR.KPC2S) == (const.SOLAR2S, const.MPC2S, const.KPC2S)
    assert DR.TWO_PI == 2 * DR.PI == 2 * np.pi and DR.LD(-5.0 / 3) != DR.LD(-5) / DR.LD(3)


# ------------------------------------------------------------------ the bounds reject wrong results
def _rejects(dev, ref, check=DR.check):
    try:
        check(dev, ref)
    except AssertionError:
        return True
    return False


def test_fourier_mutants_rejected():
    for kind, conv, muts in (("gen", 1, ("swap", "row_shift")), ("gen", 0, ("row_shift",)), ("own", 0, ("nbr_freq",)),
                             ("own", 1, ("swap", "nbr_freq"))):
        b = DR.fourier_batch(kind, 10, conv, plan_only=True)
        pl = b.plan()
        ref = DR.ftile(pl, b.t0_table, conv)
        DR.check(DR.ftile(pl, b.t0_table, conv, DR.NK), ref, f"{kind} conv {conv}")       # fp64 numpy passes
        for m in muts:
            assert _rejects(DR.ftile(pl, b.t0_table, conv, DR.NK, (m,)), ref), (kind, conv, m)


def test_cholesky_mutants_rejected():
    rng = np.random.default_rng(3)
    for n in (2, 33, 67):
        A = DR.spd(n, 1e4, rng)
        A = A * 3.0                                               # l_jj far from 1
        ref = DR.cholesky_ref(A, DR.cholesky_np(A))
        DR.check(A, ref)
        for m in ("nodiv_last", "no_sqrt"):
            L = DR.cholesky_np(A, (m,))
            assert _rejects(A, DR.cholesky_ref(A, L)), (n, m)


def test_prefactor_mutants_rejected():
    cat = DR.catalog(257, seed=5)
    phat = DR.phat_of(1.0, 0.3)
    for use_pphase in (0, 1):
        ref = DR.pre_ref(cat, phat, 1.2, 1.5, use_pphase)
        DR.check_nan(DR.prefactors_np(cat, phat, 1.2, 1.5, use_pphase), ref)
        for m in ("phase0_full", "swap_fpc"):
            dev = DR.prefactors_np(cat, phat, 1.2, 1.5, use_pphase, (m,))
            assert _rejects(dev, ref, DR.check_nan), (use_pphase, m)


CW_MUTANTS = ("psr_sign", "tp_plus", "cbrt_omega", "exact53")


def _cgw_case(b, src, mode, psr):
    a = b.cgw_inputs(*src[:8], pdist=np.linspace(0.5, 2.0, b.n_psr), psrTerm=bool(psr), evolve=mode == 0,
                     phase_approx=mode == 1, tref=src[8])
    sel = np.concatenate([np.arange(o, o + n) for o, n in zip(b.toa_off, b.ntoa)])
    return a, sel


def test_cw_mutants_rejected_single_source_and_catalog():
    from tests import generator_reference as GR
    b = GR.gen_batch(red=0, white=False, ecorr=False, plan_only=True)
    sources = DR.CGW_SOURCES + (DR.near_merger(np.concatenate(b.mjd)),)
    caught = {m: [] for m in CW_MUTANTS}
    for si, src in enumerate(sources):
        for mode in (0, 1, 2):
            for psr in (0, 1):
                a, sel = _cgw_case(b, src, mode, psr)
                ref = DR.cgw_ref(a, sel=sel).out()
                DR.check(DR.cgw_ref(a, DR.NK, sel=sel), ref, f"cgw {si} {mode} {psr}")
                for m in CW_MUTANTS:
                    if _rejects(DR.cgw_ref(a, DR.NK, (m,), sel=sel), ref):
                        caught[m].append((si, mode, psr))
    assert all(caught.values()), {m: len(v) for m, v in caught.items()}
    # the same mutants through a catalog sum: one-source catalogs of the sweep's sources (a sum over many sources adds
    # their bounds, which hides the exponent mutant) and a 300-source catalog
    t = DR.cat_toas(129, seed=8)
    phat = DR.phat_of(2.0, -0.4)
    cats = [np.array(src[:8], dtype=float)[:, None] for src in DR.CGW_SOURCES if src[8] == 53000 * 86400.0]
    cats.append(DR.catalog(300, seed=8, merged=0.0))
    caught = {m: 0 for m in CW_MUTANTS}
    for cat in cats:
        for tag in ("evolve", "approx", "mono", "earth"):
            mode, psr, pdist, pph, use = DR.cat_variant(tag)
            pre = DR.prefactors_np(cat, phat, pdist, pph, use)
            ref, rs = DR.catalog_sum_ref(pre, t, mode, psr)
            DR.check(DR.catalog_sum_np(rs, 2), ref, tag)
            q = [pre[:, k][:, None] for k in range(14)]
            for m in CW_MUTANTS:
                r = DR.cw_res(DR.NK, t[None, :], q, mode, psr, (m,))
                caught[m] += _rejects(DR.catalog_sum_np(r, 2), ref)
    assert all(caught.values()), caught


def test_catalog_summation_mutants_rejected():
    cat = DR.catalog(257, seed=9, merged=0.2)
    t = DR.cat_toas(129, seed=9)
    pre = DR.prefactors_np(cat, DR.phat_of(0.4, 0.9), 1.2, 0.0, 0)
    ref, rs = DR.catalog_sum_ref(pre, t, 0, 1)
    assert np.isnan(rs).any(axis=0).all() and np.isfinite(rs).any(axis=0).all()
    for ns in (2, 3, 64):
        DR.check(DR.catalog_sum_np(rs, ns), ref, f"{ns} slices")
        for m in ("drop32", "twice", "nan") if ns < 8 else ("twice", "nan"):     # 64 slices of 257: no 32-source stage
            assert _rejects(DR.catalog_sum_np(rs, ns, mut=(m,)), ref), (ns, m)


# ------------------------------------------------------------------ the sweep reaches its edges
def test_sweep_reaches_the_kernel_edges():
    from tests import generator_reference as GR
    b = GR.gen_batch(red=10, white=False, ecorr=False, plan_only=True)
    tl = b.plan()["tiles"]
    nep = set(tl[:, 4].tolist())
    assert {16, 17, 32, 33, 64} <= nep
    # an epoch split across two tiles: the next tile of the same pulsar starts at this tile's last epoch
    split = [(k, k + 1) for k in range(len(tl) - 1) if tl[k, 5] == tl[k + 1, 5] and tl[k + 1, 3] == tl[k, 3] + tl[k, 4] - 1]
    assert split
    # nrows K crosses a 256-thread block mid-row for some swept K
    nrows = int(tl[:, 4].sum())
    assert any(256 % K and nrows * K > 256 for K in DR.FOURIER_K)
    # the per-pulsar-Tspan batch: different frequencies per pulsar, and conv = 0 arguments from < 1e3 to > 1e9 rad
    bo = DR.fourier_batch("own", 2, 0, plan_only=True)
    plo = bo.plan()
    f = plo["freqs"]
    assert len(np.unique(f[:, 0])) == bo.n_psr
    _, _, pp, tt = DR.fourier_rows(plo, bo.t0_table, 0)
    arg = 2 * np.pi * tt[:, None] * f[pp]
    assert arg.min() < 1e3 and arg.max() > 1e9 and np.any((arg > 1e5) & (arg < 1e8))
    # catalogs: stages ending at cnt < 32, more than one slice, unequal slices, empty slices
    stage_ends, multi, unequal, empty = set(), False, False, False
    for n_src, spec, n_toa, _, _ in DR.CAT_CASES:
        ls = DR.slice_lengths(n_src, DR.n_slices_of(n_src, spec))
        stage_ends |= {x % 32 for x in ls if x}
        nz = [x for x in ls if x]
        multi |= len(nz) > 1
        unequal |= len(set(nz)) > 1
        empty |= 0 in ls
    assert stage_ends - {0} and 0 in stage_ends and multi and unequal and empty
    toas = {c[2] for c in DR.CAT_CASES}
    assert {1, 127, 128, 129, 1025} <= toas and {1, 31, 32, 33, 256, 257, 4097, 16385} <= {c[0] for c in DR.CAT_CASES}
    assert {DR.cat_variant(c[3]) for c in DR.CAT_CASES} == {DR.cat_variant(t) for t in ("evolve", "earth", "approx", "mono",
                                                                                        "pphase")}
    # the toa sample of a large catalog holds each CTA's first and last TOA
    idx = DR.toa_sample(1025, 16385, np.random.default_rng(0))
    assert {0, 127, 128, 255, 1023, 1024} <= set(idx.tolist()) and len(idx) <= 45


def test_ng15_sky_replay_matches_the_synthetic_pulsars():
    from pta_replicator_b200 import orf as orf_mod
    from pta_replicator_b200 import synthetic
    psrs, _ = synthetic.make_ng15_like("epoch", npsr=5)
    assert np.array_equal(DR.ng15_radec("epoch", npsr=5), orf_mod.psrlocs_from_pulsars(psrs))
    assert DR.ng15_radec("full").shape == (67, 2)
