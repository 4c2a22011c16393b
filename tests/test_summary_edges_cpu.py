"""CPU tests of the extended-precision reference of the summary kernels (tests/summary_reference.py): closed forms, the
fp64 oracle the GPU tests trust (``curn_oracle.summaries``) and the fp64 restatement of ``fp_q_int`` against it on the
constructed families the GPU sweep uses, every mutant rejected by a constructed case, and the engine's trapezoid
weights and prior against the restatement."""
import numpy as np
import pytest

from tests import curn_oracle as CO
from tests import reduction_reference as RR
from tests import summary_reference as SR

U = RR.U
pytestmark = pytest.mark.skipif(not RR.LONG, reason="the reference needs a 64-bit mantissa longdouble")


def _ref(maps, x, g, kind, ul, mutant=None):
    st = SR.statics(x, g, kind)
    return SR.curn_summaries(maps, x, g, st["wg"], st["wx"], st["prior"], ul, mutant), st


# ------------------------------------------------------------------ closed forms
@pytest.mark.parametrize("spacing", SR.SPACINGS)
@pytest.mark.parametrize("kind", SR.PRIORS)
def test_constant_map(spacing, kind):
    x, g = SR.grid(64, 5, spacing)
    for c in (0.0, -3.25, 1e300):
        ref, st = _ref(np.full((1, 5, 64), c), x, g, kind, 0.95)
        wgs = float(SR.trapezoid_weights(g).sum())
        assert abs(ref["ln_bayes"]["hi"][0] - c) <= 1e-15 * max(1.0, abs(c))
        np.testing.assert_allclose(ref["post_log10_A"]["hi"][0], st["prior"] * wgs, rtol=1e-15)
        np.testing.assert_allclose(ref["post_gamma"]["hi"][0], 1 / wgs, rtol=1e-15)
        assert ref["lnL_max"][0] == c and ref["ml_gamma_index"][0] == 0 and ref["ml_log10_A_index"][0] == 0
        if kind == "log-uniform":
            for ul in SR.ULS:
                q = SR.curn_ul(SR.curn_core(np.full((1, 5, 64), c), x, g, st["wg"], st["wx"], st["prior"]), ul)
                assert abs(q["hi"][0] - (x[0] + ul * (x[-1] - x[0]))) <= q["bound"][0] + 1e-14
                assert q["bound"][0] <= 1e-12


@pytest.mark.parametrize("spacing", ("uniform", "geometric"))
def test_single_spike(spacing):
    """A spike 1e4 above its floor: ln_bayes = m + ln(wg wx prior) at the node, the posterior is two triangles."""
    x, g = SR.grid(64, 5, spacing)
    k, j = 20, 3
    m = np.full((1, 5, 64), 2.5 - 1e4)
    m[0, j, k] = 2.5
    for ul in (0.25, 0.5, 0.95):
        ref, st = _ref(m, x, g, "uniform", ul)
        assert abs(ref["ln_bayes"]["hi"][0] - (2.5 + np.log(st["wg"][j] * st["wx"][k] * st["prior"][k]))) <= 1e-14
        d0, d1 = x[k] - x[k - 1], x[k + 1] - x[k]
        q = x[k - 1] + ul * (d0 + d1) if ul * (d0 + d1) <= d0 else x[k] + (ul * (d0 + d1) - d0)
        assert abs(ref["log10_A_ul"]["hi"][0] - q) <= ref["log10_A_ul"]["bound"][0] + 1e-14
        assert ref["log10_A_ul"]["bound"][0] <= 1e-10
        assert (ref["ml_gamma_index"][0], ref["ml_log10_A_index"][0]) == (j, k)


def test_uniform_in_A_prior_against_the_analytic_integral():
    x, g = SR.grid(256, 1, "uniform")
    p = SR.prior_density(x, g, "uniform").astype(float)
    a = 10.0 ** x
    np.testing.assert_allclose(p, a * np.log(10) / (a[-1] - a[0]), rtol=1e-3)   # trapezoid error (ln 10 dx)^2 / 12
    ref, _ = _ref(np.zeros((1, 1, 256)), x, g, "uniform", 0.95)
    assert abs(ref["log10_A_ul"]["hi"][0] - np.log10(a[0] + 0.95 * (a[-1] - a[0]))) <= 2e-3


def test_first_max_rule():
    nan, inf = np.nan, np.inf
    assert SR.first_max([1, 3, 3, 2]) == 1 and SR.first_max([-inf, -inf]) == 0
    assert SR.first_max([5, nan, inf, nan]) == 1 and SR.first_max([nan]) == 0
    assert SR.first_max([1, inf, inf]) == 1 and SR.first_max([2, 2, -inf]) == 0


# ------------------------------------------------------------------ the fp64 oracle on the constructed families
@pytest.mark.parametrize("NA,NG", SR.GRIDS)
@pytest.mark.parametrize("spacing", SR.SPACINGS)
def test_fp64_oracle_within_reference_bounds(NA, NG, spacing):
    """``curn_oracle.summaries`` rounds its own weights and prior, hence the slack of 16 u on each relative bound."""
    x, g = SR.grid(NA, NG, spacing)
    names, maps = SR.curn_maps(x, g)
    worst = 0.0
    for kind in SR.PRIORS:
        st = SR.statics(x, g, kind)
        core = SR.curn_core(maps, x, g, st["wg"], st["wx"], st["prior"])
        for ul in SR.ULS:
            ref = {k: v for k, v in core.items() if not k.startswith("_")}
            ref["log10_A_ul"] = SR.curn_ul(core, ul)
            with np.errstate(all="ignore"):
                got = CO.summaries(maps, x, g, kind, ul)
            worst = max(worst, SR.curn_compare(got, ref, f"{NA}x{NG} {spacing} {kind} ul={ul}", slack=16))
    print(f"\n[summary] fp64 oracle, {NA}x{NG} {spacing}, {len(names)} maps: worst |d|/bound {worst:.3f}")


def test_reference_follows_the_non_finite_rule():
    x, g = SR.grid(64, 5, "geometric")
    names, maps = SR.curn_nonfinite_maps(x, g)
    ref, _ = _ref(maps, x, g, "log-uniform", 0.95)
    for r, name in enumerate(names):
        flat = maps[r].ravel()
        if name == "all -inf":
            assert ref["lnL_max"][r] == -np.inf and ref["ln_bayes"]["hi"][r] == -np.inf
            assert (ref["ml_gamma_index"][r], ref["ml_log10_A_index"][r]) == (0, 0)
            nanout = ("post_log10_A", "post_gamma", "log10_A_ul")
        elif name.startswith("-inf"):
            assert np.isfinite(ref["lnL_max"][r])
            assert all(np.all(np.isfinite(ref[k]["hi"][r])) for k in SR.CURN_BOUNDED)
            continue
        else:
            nanout = SR.CURN_BOUNDED
            first = np.flatnonzero(np.isnan(flat))[0] if np.isnan(flat).any() else np.flatnonzero(np.isposinf(flat))[0]
            assert ref["ml_gamma_index"][r] * 64 + ref["ml_log10_A_index"][r] == first
        assert all(np.all(np.isnan(ref[k]["hi"][r])) for k in nanout), name


# ------------------------------------------------------------------ mutants
def _rows_outside(dev, ref):
    """Per map: is any output of ``dev`` (a reference's central values) outside ``ref``'s bounds?"""
    bad = np.zeros(len(ref["lnL_max"]), dtype=bool)
    for k in SR.CURN_EXACT:
        bad |= ~((dev[k] == ref[k]) | (np.isnan(dev[k].astype(float)) & np.isnan(ref[k].astype(float))))
    for k in SR.CURN_BOUNDED:
        a, h = dev[k]["hi"], ref[k]["hi"]
        with np.errstate(invalid="ignore"):
            ok = (np.abs((a - h) - ref[k]["lo"]) <= ref[k]["bound"]) | (np.isnan(a) & np.isnan(h)) | (a == h)
        bad |= ~(ok.reshape(len(bad), -1).all(axis=1))
    return bad


def _mutant_cases():
    for NA, NG, spacing, kind, ul in ((3, 2, "uniform", "log-uniform", 0.5), (64, 5, "geometric", "uniform", 0.95),
                                      (64, 5, "uniform", "log-uniform", 0.5), (97, 57, "tiny", "log-uniform", 1e-6)):
        x, g = SR.grid(NA, NG, spacing)
        n1, m1 = SR.curn_maps(x, g)
        n2, m2 = SR.curn_nonfinite_maps(x, g)
        yield f"{NA}x{NG} {spacing} {kind} ul={ul:g}", x, g, kind, ul, n1 + n2, np.concatenate([m1, m2])


def test_every_mutant_is_rejected_by_a_constructed_case():
    killed, lines = {}, []
    cases = list(_mutant_cases())
    refs = [_ref(maps, x, g, kind, ul)[0] for _, x, g, kind, ul, _, maps in cases]
    for (tag, x, g, kind, ul, names, maps), ref in zip(cases, refs):
        assert not _rows_outside(ref, ref).any()
    for mu in SR.MAX_MUTANTS + SR.CURN_MUTANTS:
        for (tag, x, g, kind, ul, names, maps), ref in zip(cases, refs):
            bad = _rows_outside(_ref(maps, x, g, kind, ul, mu)[0], ref)
            if bad.any():
                killed[mu] = f"{tag}: {names[int(np.argmax(bad))]} (+ {int(bad.sum()) - 1} more)"
                break
        lines.append(f"{mu:>16s}: {killed.get(mu, 'SURVIVES')}")
    # Fp: Q(P, x) and the maxima
    for mu in SR.FP_MUTANTS:
        for P in (1, 2, 16, 17, 67):
            xs = SR.fp_x_values(P)
            q, qb = SR.q_ref(P, xs)
            qm, _ = SR.q_ref(P, xs, mu)
            with np.errstate(invalid="ignore"):
                bad = np.abs((qm - q).astype(float)) > qb
            if bad.any():
                killed[mu] = f"Q({P}, x = {xs[int(np.argmax(bad))]!r})"
                break
        lines.append(f"{mu:>16s}: {killed.get(mu, 'SURVIVES')}")
    fm = np.array([[1.0, 4.0, 4.0, np.nan, 2.0, np.nan]])
    for mu in SR.MAX_MUTANTS:
        good, wrong = SR.fe_combine(fm[:, :3] if mu == "tie_high" else fm, np.arange(6)[None]), None
        wrong = SR.fe_combine(fm[:, :3] if mu == "tie_high" else fm, np.arange(6)[None], mu)
        assert good["argmax_f"][0] != wrong["argmax_f"][0], mu
    print("\n[summary] mutant -> the first constructed case that rejects it:\n  " + "\n  ".join(lines))
    assert set(killed) == set(SR.MAX_MUTANTS + SR.CURN_MUTANTS + SR.FP_MUTANTS), lines


# ------------------------------------------------------------------ Q(P, x)
@pytest.mark.parametrize("P", (1, 2, 15, 16, 17, 67, 128))
def test_fp64_q_int_within_the_stated_error(P):
    """The fp64 restatement of fp_q_int (``RR.q_int``) against mpmath over the branch sweep: relative error within
    Q_CONST (x + P) 2^-53 (plus 4 subnormal ulps), the bound the GPU test holds the device to."""
    xs = SR.fp_x_values(P)
    q, qb = SR.q_ref(P, xs)
    with np.errstate(all="ignore"):
        got = RR.q_int(P, xs)
        ratio = np.abs((got.astype(SR.LD) - q).astype(float)) / qb
    print(f"\n[summary] fp64 q_int P={P}: worst |d|/bound {np.nanmax(ratio):.3f} at x = {xs[int(np.nanargmax(ratio))]!r}")
    assert np.all(ratio <= 1.0)
    assert got[0] == 1.0 and got[-1] == 0.0


def test_fp_amps_construct_the_chosen_values_exactly():
    for P in (1, 17, 128):
        xs = SR.fp_x_values(P)
        a = SR.fp_amps_of(xs, P, 2)
        ref = SR.fp_summaries(a, P)
        fin = np.isfinite(xs)
        for f in range(2):
            want = xs[(np.arange(len(xs)) + f) % len(xs)]
            assert np.array_equal(ref["Fp"]["hi"][:, f], want) and np.all(ref["Fp"]["lo"][:, f][fin] == 0)


# ------------------------------------------------------------------ the engine's statics
@pytest.mark.parametrize("spacing", ("geometric", "tiny"))
def test_engine_weights_and_prior_match_the_restatement(spacing):
    from pta_replicator_b200 import engine
    from tests.test_optimal_statistic_cpu import _batch, _small
    x, g = SR.grid(64, 5, spacing)
    for v in (x, g, g[:1], x[:2]):
        np.testing.assert_allclose(engine._trapezoid_weights(v), SR.trapezoid_weights(v).astype(float), rtol=4 * U, atol=0)
    b = _batch(_small())
    for kind in SR.PRIORS:
        b.set_curn_likelihood(log10_A=x, gamma=g, components=3, amplitude_prior=kind)
        pc = b.plan()["curn"]
        st = SR.statics(x, g, kind)
        np.testing.assert_allclose(pc["wg"], st["wg"], rtol=4 * U)
        np.testing.assert_allclose(pc["wx"], st["wx"], rtol=4 * U)
        np.testing.assert_allclose(pc["prior"], st["prior"], rtol=2e-14)        # 10^x in fp64: |x ln 10| u on each node
