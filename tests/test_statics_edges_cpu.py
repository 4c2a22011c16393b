"""CPU tests of the statistics' host statics (``plan()``: optimal statistic, anisotropy, Fp, Fe, CURN, HD) at edge noise
recipes against the extended-precision dense reference of tests/statics_reference.py: the statics applied in numpy to
a few rows (the eigen forms the kernels evaluate) against the definitions evaluated in long double and mpmath.

Tolerances are relative to the scale of the terms: |d ln L| <= TAU (1 + Q/2 + ldet/2) for CURN and HD, |d rho| <= TAU
|x_a||x_b| / t_ab and its template sums for the optimal statistic, |d Fp| <= TAU Fp, |d X^| <= TAU max(1, |X^|),
|d Fe| <= TAU max(1, Fp), the same |x_a||x_b| sums for the anisotropy fits and the radiometer; the statics C and Z
against TAU max|C_a|, TAU max|Z_a|.  Where a recipe is ill-conditioned the tolerance grows with the condition number
the reference reports (``_tau``).  Every case prints its worst |d| / tolerance per output and the condition numbers."""
import numpy as np
import pytest

from tests import curn_oracle as CO
from tests import hd_oracle as HO
from tests import statics_reference as SR

TAU = 1e-10
# CURN and HD: the eigen form phi~^1/2 Z phi~^1/2 = U diag(lambda) U^T carries absolute eigenvalue errors ~u lambda_max
# (LAPACK), and at gamma = 7 with K = 16 phi~ alone spans 16^7; the loud corners weigh the small eigenvalues in.
TAU_LIKE = 1e-9
RECIPES = SR.recipes()
# Recipes where the statics are outside TAU_LIKE (a finding, recorded here until the eigen form or the PSD refusal is
# reworked): the measured worst |d| / (TAU_LIKE scale) is in the reason.
# (recipe, statistic) -> (outputs, kind, what): discrepancies of the plan's CURN / HD statics beyond TAU_LIKE, each with
# the explanation the test demonstrates --
#   "eigen": tier 2 evaluated on the plan's own C (no eigendecomposition) is within TAU_LIKE, so the error is the fp64
#            eigen form, whose eigenvalues carry absolute errors ~u lambda_max while the loud corners weigh the small ones;
#   "zcond": Z_a is right to rounding normwise (|dZ_a| / |Z_a|, measured) but ill-conditioned, and the relative error
#            of ln L is within 2K max_a |dZ_a| / |Z_a| kappa(Z_a), the first-order trace bound of
#            d ln det(I + A^2 Zh) = tr((I + A^2 Zh)^-1 A^2 dZh) over 2K directions at the loud corners;
#   "woodbury": the eigen-free evaluation of the plan's C is off by as much, and the relative error is within
#            u max(kappa(S), kappa_c), the first-order bound of the fp64 Woodbury form and the cancellation of N^-1 F by
#            the red-noise and timing-model terms (``SR.cancellation_cond``).
KNOWN = {
    ("corners_k16_hd", "hd"): (("hd lnL", "hd ldet"), "eigen", "gamma = 7, K = 16, N = 64"),
    ("orf_rank2", "hd"): (("hd lnL",), "eigen", "rank-2 ORF"),
    ("rankdef", "curn"): (("curn lnL", "curn ldet"), "eigen", "n_a = 5, 6, 7 < 2K = 32"),
    ("chrom_dm_only_rn", "curn"): (("curn lnL", "curn ldet"), "eigen", "loud DM noise, gamma = 7 at log10_A = -11"),
    ("red_gw_modes", "curn"): (("curn lnL", "curn ldet"), "woodbury", "loud red noise on the GW frequencies"),
    ("red_loud", "curn"): (("curn lnL", "curn ldet"), "woodbury", "loud steep red noise, 30 components"),
    ("red_loud_hd", "curn"): (("curn lnL", "curn ldet"), "woodbury", "loud steep red noise, K = 1"),
    ("red_loud_hd", "hd"): (("hd lnL", "hd ldet"), "woodbury", "loud steep red noise, K = 1, dipole"),
    ("tspan_2", "curn"): (("curn lnL", "curn ldet"), "zcond", "Tspan = 2 x span"),
    ("white_span", "curn"): (("curn lnL", "curn ldet"), "zcond", "sigma from 1e-8 s to 1e-5 s"),
    ("rankdef_tm", "curn"): (("curn C", "curn Z"), "woodbury", "offset + jumps leave 2-4 of 5-7 TOAs"),
    ("rankdef_tm", "os"): (("os rho", "os A2", "os snr", "os A2_mc", "os t_ab", "os C", "os Z"), "woodbury",
                           "offset + jumps leave 2-4 of 5-7 TOAs"),
    ("rankdef_hd", "curn"): (("curn C", "curn Z"), "woodbury", "offset + jumps leave 2-4 of 5-7 TOAs"),
}


def _tau(kappa, tau=TAU):
    """``tau``, grown by the condition number ``kappa`` of the system the output depends on once 64 u kappa passes it."""
    return max(tau, 64 * 2.0 ** -53 * kappa)


def _ratio(got, ref, scale, tau):
    return float(np.max(np.abs(np.asarray(got) - ref) / (tau * np.asarray(scale))))


# ------------------------------------------------------------------ the statics applied in numpy
def os_of_statics(b, po, rows):
    """rho [R, q], A2, snr, A2_mc [R, n_orf] and d [R, q] from ``plan()["os"]``."""
    nc = po["nc"]
    X = np.stack([rows[:, s:s + n] @ po["C"][s:s + n, :nc] for s, n in zip(b.toa_off, b.ntoa)], axis=1)
    x = X * po["sqrt_phi"][:nc]
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    d = np.einsum("rqj,rqj->rq", x[:, pa], x[:, pb])
    bo = d @ po["orf"].T
    return dict(rho=d / po["t_ab"], A2=bo / po["dnorm"], snr=bo / po["dsqrt"], A2_mc=bo @ po["finv"].T, d=d)


def aniso_of_statics(pa, d):
    """clm [R, n_lm], chi2 [R], radio [R, S] from ``plan()["os_aniso"]`` and the pair correlations d."""
    y = d @ pa["V"][:pa["n_col"], :pa["kd"]].T / pa["dsqrt"]
    nl, nz = pa["n_lm"], pa["n_z"]
    return dict(clm=y[:, :nl], chi2=np.sum(y[:, nl:nl + nz] ** 2, axis=1), radio=y[:, nl + nz:])


def fp_of_statics(b, pf, rows):
    """X^ [R, P, Nf, 2] and Fp [R, Nf] from ``plan()["fp"]``."""
    from pta_replicator_b200.engine import fp_whitened_basis
    amps = np.stack([rows[:, s:s + n] @ fp_whitened_basis(pf, s, n) for s, n in zip(b.toa_off, b.ntoa)], axis=1)
    amps = amps.reshape(rows.shape[0], b.n_psr, pf["n_freq"], 2)
    return amps, 0.5 * np.sum(amps ** 2, axis=(1, 3))


def fe_of_statics(pe, amps):
    """Fe [R, Nf, S] from ``plan()["fe"]`` on X^: N_a = L_a X^_a, N4 = sum_a e_a (x) N_a, Fe = 1/2 |L4^-1 N4|^2."""
    Lf, ant, S = pe["Lf"], pe["antenna"], pe["n_sky"]
    N = np.stack([Lf[None, :, :, 0].transpose(0, 2, 1) * amps[..., 0],
                  Lf[None, :, :, 1].transpose(0, 2, 1) * amps[..., 0] + Lf[None, :, :, 2].transpose(0, 2, 1) * amps[..., 1]],
                 axis=-1)                                                              # [R, P, Nf, 2]
    N4 = np.einsum("asp,rafc->rfspc", ant, N).reshape(amps.shape[0], amps.shape[2], S, 4)
    Linv = np.zeros(pe["linv"].shape[:2] + (4, 4))
    Linv[..., np.tril_indices(4)[0], np.tril_indices(4)[1]] = pe["linv"]
    y = np.einsum("fsij,rfsj->rfsi", Linv[:, :S], N4)
    return 0.5 * np.sum(y * y, axis=-1)


# ------------------------------------------------------------------ cases
def _kappa(e, common=None, own_red=True):
    """The largest kappa of the pulsars' Woodbury matrices S (chromatic blocks included; the red noise left out with
    ``own_red`` False) and of their ECORR Sherman-Morrison steps (1 + e^2 sum_bucket 1/sigma^2, the cancellation of
    N^-1 V within a bucket)."""
    b = e.b
    k = max(SR.woodbury_cond(b, i, common, e.tm[i], own_red) for i in range(b.n_psr))
    if b._ecorr is not None:
        for i in range(b.n_psr):
            bucket, ec = b._ecorr[i]
            w1, w2 = b._white[i]
            k = max(k, float(np.max(1 + np.asarray(ec)[bucket] ** 2 * np.bincount(bucket, 1 / (w1 * w1 + w2 * w2))[bucket])))
    return k


def _statics_ratio(b, Cplan, Zplan, ref, tau):
    """Worst |d C_a| / (tau max|C|) and |d Z_a| / (tau max|Z|) over the pulsars, max over the array: a pulsar whose
    timing model leaves a few TOAs has C_a and Z_a 1e17 below its unprojected P_a^-1 F and F^T P_a^-1 F, which no fp64
    evaluation resolves, and contributes accordingly little to every statistic."""
    Cs = [c.astype(np.float64) for c in ref["C"]]
    cmax, zmax = max(np.max(np.abs(c)) for c in Cs), np.max(np.abs(ref["Z"]))
    rc = max(_ratio(Cplan[s:s + n, :C.shape[1]], C, cmax, tau) for C, s, n in zip(Cs, b.toa_off, b.ntoa))
    return rc, _ratio(Zplan, ref["Z"], zmax, tau)


STATS = ("curn", "hd", "os", "aniso", "fp", "fe")


def cases():
    """(recipe, statistic) for every statistic a recipe registers."""
    out = []
    for name in sorted(RECIPES):
        st = RECIPES[name]().stats
        out += [(name, k) for k in STATS if k in st]
    return out


def e_nc(name):
    return RECIPES[name]().stats["curn"]["K"]


def _ncols(e, i):
    M = SR.design(e.b, i, e.tm[i])
    return 0 if M is None else M.shape[1]


def _plan_C(b, pl, nc):
    return [pl["C"][s:s + n, :nc] for s, n in zip(b.toa_off, b.ntoa)]


def run_case(name, stat):
    """Statistic ``stat`` of recipe ``name``: ({output: worst |d| / tolerance}, the conditions used, {output: worst
    |d| / tolerance of the eigen-free evaluation of the plan's own C (CURN, HD only)})."""
    e = RECIPES[name]()
    b = e.b
    pl = b.plan()
    rows = SR.rows_of(b, 3, seed=len(name))
    out, cond, free = {}, {}, {}
    kap = _kappa(e)
    cond["S"] = kap
    tau = _tau(kap)
    if stat in ("curn", "hd"):
        pc = pl["curn"]
        if stat == "curn":
            ref = SR.curn(e, rows)
            out["curn lnL"] = _ratio(CO.lnl_of_statics(b, pc, rows), ref["lnl"], ref["scale"], TAU_LIKE)
            out["curn ldet"] = _ratio(pc["ldet"], ref["ldet"], 1 + ref["ldet"], TAU_LIKE)
            out["curn C"], out["curn Z"] = _statics_ratio(b, pc["C"], pc["Z"], ref, tau)
            full = [i for i in range(b.n_psr) if b.ntoa[i] - _ncols(e, i) >= pc["nc"]]      # Z_a of full rank
            ev = np.linalg.eigvalsh(ref["Z"][full]) if full else np.ones((1, 1))
            dz = [np.max(np.abs(pc["Z"][i] - ref["Z"][i])) / np.max(np.abs(ref["Z"][i])) for i in full] or [0.0]
            cond["Z_a"] = float(np.max(ev[:, -1] / ev[:, 0]))
            cond["dZ kappa(Z_a)"] = float(np.max(np.array(dz) * ev[:, -1] / ev[:, 0]))
            own = SR.curn(e, rows, given=_plan_C(b, pc, pc["nc"]))
            free["curn lnL"] = _ratio(own["lnl"], ref["lnl"], ref["scale"], TAU_LIKE)
        else:
            rh = SR.hd(e, rows)
            out["hd lnL"] = _ratio(HO.lnl_of_statics(b, pc, pl["hd"], rows), rh["lnl"], rh["scale"], TAU_LIKE)
            out["hd ldet"] = _ratio(pl["hd"]["ldet"], rh["ldet"], 1 + rh["ldet"], TAU_LIKE)
            own = SR.hd(e, rows, given=_plan_C(b, pc, pc["nc"]))
            free["hd lnL"] = _ratio(own["lnl"], rh["lnl"], rh["scale"], TAU_LIKE)
    elif stat in ("os", "aniso"):
        o = e.stats["os"]
        if o["log10_A_common"] is not None:
            kap = max(SR.woodbury_cond(b, i, _common_gw(e, i), e.tm[i]) for i in range(b.n_psr))
            cond["S (os, common)"] = kap
            tau = _tau(kap)
        po = pl["os"]
        got = os_of_statics(b, po, rows)
        if stat == "os":
            ref = SR.optimal_statistic(e, rows)
            for k in ("rho", "A2", "snr", "A2_mc"):
                out[f"os {k}"] = _ratio(got[k], ref[k], ref[k + "_s"], tau)
            out["os t_ab"] = _ratio(po["t_ab"], ref["t_ab"], ref["t_ab"], tau)
            out["os C"], out["os Z"] = _statics_ratio(b, po["C"], po["Z"], ref, tau)
        else:
            an = pl["os_aniso"]
            ra = SR.anisotropy(e, rows, an.get("T_sph"))
            ga = aniso_of_statics(an, got["d"])
            if "clm" in ra:
                out["aniso clm"] = _ratio(ga["clm"], ra["clm"], ra["clm_s"], tau)
                out["aniso chi2"] = _ratio(ga["chi2"], ra["chi2"], 1 + ra["chi2_s"], tau)
            if "radio" in ra:
                out["aniso radio"] = _ratio(ga["radio"], ra["radio"], ra["radio_s"], tau)
    else:
        o = e.stats["fp"]
        if o["log10_A_common"] is not None:
            kap = max(SR.woodbury_cond(b, i, _common_fp(e, i), e.tm[i]) for i in range(b.n_psr))
            cond["S (fp, common)"] = kap
            tau = _tau(kap)
        rf = SR.fp(e, rows)
        cond["M_a(f)"] = float(rf["kappa"].max())
        amps, Fp = fp_of_statics(b, pl["fp"], rows)
        if stat == "fp":
            out["fp X^"] = _ratio(amps, rf["amps"], np.maximum(1, np.abs(rf["amps"])), tau)
            out["fp Fp"] = _ratio(Fp, rf["Fp"], rf["Fp"], tau)
            out["fp M"] = _ratio(pl["fp"]["M"], rf["M"], np.max(np.abs(rf["M"]), axis=(2, 3))[..., None, None], tau)
        else:
            rfe = SR.fe(e, rows, rf)
            cond["M4"] = float(rfe["kappa"].max())
            out["fe Fe"] = _ratio(fe_of_statics(pl["fe"], amps), rfe["Fe"], np.maximum(1, rf["Fp"])[:, :, None], tau)
    return out, cond, free


def _common_gw(e, i):
    o = e.stats["os"]
    T = SR.array_tspan(e.b, o["Tspan"])
    f = np.arange(1, o["K"] + 1) / T
    return SR.basis(e.b.t_tdb[i], f), SR.ld_phi(f, o["gamma"], T, o["log10_A_common"])


def _common_fp(e, i):
    o = e.stats["fp"]
    T = SR.array_tspan(e.b, o["Tspan"])
    f = np.arange(1, o["components_common"] + 1) / T
    return SR.basis(e.b.t_tdb[i], f), SR.ld_phi(f, o["gamma_common"], T, o["log10_A_common"])


@pytest.mark.skipif(not SR.LONG, reason="the statics reference needs an 80-bit long double")
def test_reference_self_check():
    """Tier 1 in long double against tier 1 entirely in mpmath on the smallest recipe (5 TOAs, K = 16).  With a timing
    model that leaves 2 of 5 TOAs the long-double path loses to the constrained form's cancellation (printed), which is
    why tier 1 runs in mpmath for pulsars of at most MP_TOAS TOAs."""
    d = SR.self_check(RECIPES["rankdef"]())
    dt = SR.self_check(RECIPES["rankdef_tm"]())
    print(f"\n[statics reference] long double vs mpmath tier 1, max |d C| / max |C|: {d:.1e} (rankdef), {dt:.1e} "
          f"(rankdef_tm, long double path; the reference uses mpmath below {SR.MP_TOAS + 1} TOAs)")
    assert d <= 1e-15


@pytest.mark.skipif(not SR.LONG, reason="the statics reference needs an 80-bit long double")
@pytest.mark.parametrize("name,stat", cases())
def test_statics_against_extended_precision(name, stat):
    out, cond, free = run_case(name, stat)
    print(f"\n[statics edges] {name} / {stat}: TAU {TAU:.0e}, TAU_LIKE {TAU_LIKE:.0e}, conditions " +
          ", ".join(f"kappa({k}) {v:.1e}" for k, v in cond.items()))
    for k, v in out.items():
        print(f"    {k:>12s}: worst |d| / tolerance {v:.3g}" + (f"  (eigen-free on the plan's C: {free[k]:.3g})"
                                                                 if k in free else ""))
    known, kind, _ = KNOWN.get((name, stat), ((), None, ""))
    bad = {k: v for k, v in out.items() if not v <= 1.0 and k not in known}
    assert not bad, f"{name}: outside tolerance {bad}"
    if kind is None:
        return
    assert any(not out[k] <= 1.0 for k in known), f"{name} {stat}: the recorded discrepancy is gone, remove it from KNOWN"
    f = free.get(stat + " lnL", np.inf)
    if kind == "eigen":
        assert f <= 1.0, f"{name} {stat}: the plan's C evaluated without the eigen form is off too ({f:.3g})"
    elif kind == "zcond":
        allow = 2 * e_nc(name) * cond["dZ kappa(Z_a)"] / TAU_LIKE
        print(f"    2K max_a |dZ_a| / |Z_a| kappa(Z_a) (full-rank pulsars) = {allow:.3g} x TAU_LIKE")
        assert f > 1.0 and max(out[k] for k in known) <= allow, f"{name} {stat}: not Z's conditioning"
    else:
        e = RECIPES[name]()
        o = e.stats["os" if stat == "os" else "curn"]
        kc = SR.cancellation_cond(e, o["K"], SR.array_tspan(e.b, o["Tspan"]))
        allow = 2.0 ** -53 * max(cond["S"], kc) / TAU_LIKE
        print(f"    kappa_c {kc:.1e}: u max(kappa(S), kappa_c) = {allow:.3g} x TAU_LIKE")
        lnl_known = stat + " lnL" in known
        assert (f > 1.0 or not lnl_known) and max(out[k] for k in known) <= allow, f"{name} {stat}: not the Woodbury bound"


def test_plan_refuses_what_the_statistics_cannot_define():
    """An Fp frequency the timing model absorbs (1 / Tspan against an extra column sin(2 pi t / Tspan + 1e-7)) and an
    Fe sky point inside a pulsar's FE_POLE_TOL cone of a 2-pulsar array (one pattern left: M4 has rank 2)."""
    e = SR.collinear(accept=False)
    with pytest.raises(ValueError, match="the timing model or the noise absorbs this frequency"):
        e.b.plan()
    e = SR._noise(SR.Edge("pole_inside", SR.pulsars(SR.EDGE4[-2:], 93)))
    e.fp(n_freqs=2, sky=SR.near_pole_sky(e.b, 0, 1.0e-6))
    with pytest.raises(ValueError, match="do not span both polarisations"):
        e.b.plan()


def test_antenna_patterns_near_a_line_of_sight():
    """engine.antenna_patterns at 1e-6 .. 4e-6 rad from a pulsar (the FE_POLE_TOL cone is ~1.4e-6 rad) against the
    patterns in mpmath from the same fp64 angles: zero inside the cone, 1e-10 relative outside it."""
    import mpmath as mp
    from pta_replicator_b200.engine import antenna_patterns
    e = SR._noise(SR.Edge("pole", SR.pulsars(SR.EDGE4, 93)))
    sky = np.concatenate([SR.near_pole_sky(e.b, i, r) for i in range(4) for r in (1.0e-6, 1.6e-6, 4.0e-6)])
    pos = SR._positions(e.b)
    got = antenna_patterns(np.pi / 2 - pos[:, 1], pos[:, 0], sky)
    with mp.workdps(SR.DPS):
        ref = np.array([[[float(v) for v in c] for c in row] for row in SR.m_antenna(e.b, sky)])
    d = np.max(np.abs(got - ref))
    print(f"\n[antenna near a line of sight] max |d| = {d:.1e} (max |F| {np.max(np.abs(ref)):.2f})")
    assert d <= 1e-10 * np.max(np.abs(ref))
