"""CPU tests of the red-noise likelihood's and the per-frequency optimal statistic's host statics (``plan()["rn"]``,
``["os_pf"]``) at edge noise recipes, chromatic ones included, against the extended-precision dense reference of
tests/statics_reference.py: the statics applied in numpy to a few rows against the definitions evaluated in long
double and mpmath.  The original statistics meet the ``chrom_*`` recipes in tests/test_statics_edges_cpu.py, which
runs every recipe of ``SR.recipes()``.

Tolerances and their scales are those of tests/test_statics_edges_cpu.py: |d ln L| <= TAU_LIKE (1 + Q/2 + ldet/2) for
the red-noise likelihood (per pulsar), |d ldet| <= TAU_LIKE (1 + ldet); the per-frequency outputs against TAU times
|X_a,k||X_b,k| / t_qk and its template sums; t_qk, D_ok, C_a and Z_a against TAU times their own scale.  The
tolerance grows with the condition number of the system (``_tau``), the Woodbury matrix here without the pulsar's
own red noise for the red-noise likelihood.  Every case prints its worst |d| / tolerance per output and the
condition numbers."""
import numpy as np
import pytest

from tests import rn_oracle as RO
from tests import statics_reference as SR
from tests.test_os_per_frequency_cpu import _plan_of_rows
from tests.test_statics_edges_cpu import TAU, TAU_LIKE, _common_gw, _kappa, _ratio, _statics_ratio, _tau

RECIPES = SR.recipes()
# existing recipes the newer statistics run on, with the registration each adds: rn(K) or the per-frequency OS on
# the recipe's optimal statistic
ON_EXISTING = {
    "rn": ("rankdef", "rankdef_tm", "ecorr_single", "ecorr_whole", "ecorr_loud", "ecorr_backend", "red_loud",
           "red_gw_modes", "white_span", "tspan_0.5", "tspan_2", "coincident_hd", "orf_rank2"),
    "pfos": ("rankdef", "rankdef_tm", "ecorr_single", "ecorr_whole", "ecorr_loud", "ecorr_backend", "red_loud",
             "red_gw_modes", "white_span", "common_loud", "coincident_os"),
}
RN_K = 4
# (recipe, statistic) -> (outputs, kind, what), the kinds of tests/test_statics_edges_cpu.py's KNOWN
KNOWN = {
    ("rankdef_tm", "rn"): (("rn C", "rn Z"), "woodbury", "offset + jumps leave 2-4 of 5-7 TOAs"),
    ("rankdef_tm", "pfos"): (("pfos rho", "pfos phi", "pfos snr", "pfos phi_mc", "pfos t_qk", "pfos D_ok"), "woodbury",
                             "offset + jumps leave 2-4 of 5-7 TOAs"),
    ("red_gw_modes", "pfos"): (("pfos rho",), "woodbury", "loud red noise on the GW frequencies"),
    ("red_loud", "rn"): (("rn lnL", "rn ldet"), "eigen", "gamma = 6.5 at log10_A = -11, timing model"),
    ("rn_tspan", "rn"): (("rn lnL", "rn ldet"), "eigen", "Tspan = 1.5 x span, timing model"),
    ("white_span", "rn"): (("rn lnL", "rn ldet"), "zfloor", "sigma from 1e-8 s to 1e-5 s, 7 TOAs for 2K = 8"),
}
# "zfloor" (a kind of its own): a rank-deficient Z_a whose eigenvalues span more than 1/u has its small ones below
# fp64 resolution wherever they are computed.  Demonstrated by the eigen-free evaluation of the plan's C being off as
# well (the fp64 Z_a carries the error before any eigen form), the error being within the first-order (Weyl) bound
# (2K)^2 u max A^2 lambda_max(phi~^1/2 Z_a phi~^1/2) / (1 + ldet) (printed), and, tighter, within ZFLOOR_FACTOR times
# the eigen-free error: the eigen form of that Z_a adds at most the same order again, so a regression of the statics
# beyond it still fails.
ZFLOOR_FACTOR = 4


def build(name, stat):
    e = RECIPES[name]()
    if stat == "rn" and "rn" not in e.stats:
        e.rn(RN_K)
    if stat == "pfos" and not e.stats["os"].get("pf"):
        e.pfos()
    return e


def cases():
    out = [(name, stat) for stat, names in ON_EXISTING.items() for name in names]
    for name in sorted(RECIPES):
        st = RECIPES[name]().stats
        out += [(name, k) for k in ("rn", "pfos") if (k == "rn" and "rn" in st) or (k == "pfos" and st.get("os", {}).get("pf"))]
    return out


def run_case(name, stat):
    """({output: worst |d| / tolerance}, the conditions used, {output: the same of the eigen-free evaluation of the
    plan's own C (red-noise likelihood only)})."""
    e = build(name, stat)
    b = e.b
    pl = b.plan()
    rows = SR.rows_of(b, 3, seed=len(name))
    out, cond, free = {}, {}, {}
    if stat == "rn":
        pr = pl["rn"]
        o = e.stats["rn"]
        common = None
        if o["log10_A_common"] is not None:
            T = SR.array_tspan(b)
            fc = np.arange(1, o["components_common"] + 1) / T
            common = lambda i: (SR.basis(b.t_tdb[i], fc), SR.ld_phi(fc, o["gamma_common"], T, o["log10_A_common"]))
        kap = _kappa(e, own_red=False) if common is None else \
            max(SR.woodbury_cond(b, i, common(i), e.tm[i], own_red=False) for i in range(b.n_psr))
        cond["S (own red out)"] = kap
        tau = _tau(kap)
        ref = SR.rn(e, rows)
        assert np.array_equal(pr["Tspan"], SR.rn_spans(e))
        out["rn lnL"] = _ratio(RO.lnl_of_statics(b, pr, rows), ref["lnl"], ref["scale"], TAU_LIKE)
        out["rn ldet"] = _ratio(pr["ldet"], ref["ldet"], 1 + ref["ldet"], TAU_LIKE)
        out["rn C"], out["rn Z"] = _statics_ratio(b, pr["C"], pr["Z"], ref, tau)
        lmax = np.array([[np.linalg.eigvalsh(ref["Z"][i] * sp[:, None] * sp[None, :])[-1] for sp in pr["sp"][i]]
                         for i in range(b.n_psr)])                                  # [P, Ng]
        free["weyl"] = float(np.max(pr["nc"] ** 2 * 2.0 ** -53 * pr["a2"][None, None, :] * lmax[..., None] /
                                    (1 + ref["ldet"])))
        own = SR.rn(e, rows, given=[pr["C"][s:s + n, :pr["nc"]] for s, n in zip(b.toa_off, b.ntoa)])
        free["rn lnL"] = _ratio(own["lnl"], ref["lnl"], ref["scale"], TAU_LIKE)
    else:
        po, pp = pl["os"], pl["os_pf"]
        kap = _kappa(e)
        if e.stats["os"]["log10_A_common"] is not None:
            kap = max(SR.woodbury_cond(b, i, _common_gw(e, i), e.tm[i]) for i in range(b.n_psr))
        cond["S"] = kap
        tau = _tau(kap)
        ref = SR.pfos(e, rows)
        got = _plan_of_rows(b, po, pp, rows)
        for k in ("rho", "phi", "snr", "phi_mc"):
            out[f"pfos {k}"] = _ratio(got[k], ref[k], ref[k + "_s"], tau)
        out["pfos t_qk"] = _ratio(pp["t"], ref["t"], ref["t"], tau)
        out["pfos D_ok"] = _ratio(pp["dnorm"], ref["D"], ref["D"], tau)
    return out, cond, free


@pytest.mark.skipif(not SR.LONG, reason="the statics reference needs an 80-bit long double")
def test_chromatic_reference_self_check():
    """Tier 1 with a DM process in P_a, long double against mpmath, on the smallest chromatic recipe (5 TOAs, K = 4)."""
    d = SR.self_check(RECIPES["chrom_dm_only_rn"]())
    print(f"\n[statics reference] chromatic tier 1, long double vs mpmath, max |d C| / max |C|: {d:.1e}")
    assert d <= 1e-15


@pytest.mark.skipif(not SR.LONG, reason="the statics reference needs an 80-bit long double")
@pytest.mark.parametrize("name,stat", cases())
def test_newer_statics_against_extended_precision(name, stat):
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
    elif kind == "zfloor":
        weyl = free["weyl"] / TAU_LIKE
        print(f"    (2K)^2 u A^2 lambda_max / (1 + ldet) = {weyl:.3g} x TAU_LIKE; {ZFLOOR_FACTOR} x eigen-free "
              f"{ZFLOOR_FACTOR * f:.3g}")
        worst = max(out[k] for k in known)
        assert f > 1.0 and worst <= min(weyl, ZFLOOR_FACTOR * f), f"{name} {stat}: not the fp64 resolution of Z_a"
    else:
        e = build(name, stat)
        if stat == "rn":
            kc = SR.cancellation_cond(e, e.stats["rn"]["K"], SR.rn_spans(e), own_red=False)
            ks = cond["S (own red out)"]
        else:
            o = e.stats["os"]
            kc, ks = SR.cancellation_cond(e, o["K"], SR.array_tspan(e.b, o["Tspan"])), cond["S"]
        allow = 2.0 ** -53 * max(ks, kc) / TAU_LIKE
        print(f"    kappa_c {kc:.1e}: u max(kappa(S), kappa_c) = {allow:.3g} x TAU_LIKE")
        lnl_known = stat + " lnL" in known
        assert (f > 1.0 or not lnl_known) and max(out[k] for k in known) <= allow, f"{name} {stat}: not the Woodbury bound"
