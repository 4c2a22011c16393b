"""CPU tests of the CURN likelihood's host statics (``PulsarBatch.set_curn_likelihood``, ``plan()["curn"]``) against
the dense oracle (tests/curn_oracle.py), of the grid summaries and of the argument checks.  ``plan_only`` batches: the
3 ``partim_small`` pulsars and the 4-pulsar synthetic case of the optimal-statistic tests, with and without a timing
model, with and without ECORR and red noise."""
import numpy as np
import pytest

from tests import curn_oracle as CO
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# ln L is a sum of terms of size up to ~1e3 on these grids; the eigen form (host statics) and the dense n x n solves
# (oracle) round differently.  The measured worst absolute difference is stated in DESIGN section 5; the bound is the
# one the likelihood must meet to serve maximum-likelihood and Bayes-factor work.
TOL = 1e-6
X_GRID = np.linspace(-15.5, -13.0, 6)
G_GRID = np.array([2.0, 13.0 / 3.0, 6.5])


def _rows(b, R, seed=0):
    """Engine-order rows [R, ld]: white draws at the TOA uncertainties plus a slow sinusoid (so that the maximum sits
    inside the grid), zero in the alignment slots."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((R, b.ld))
    for i in range(b.n_psr):
        s, n, t = b.toa_off[i], b.ntoa[i], b.t_tdb[i]
        span = np.ptp(np.concatenate(b.t_tdb))
        rows[:, s:s + n] = rng.standard_normal((R, n)) * 2e-6 + 3e-7 * np.sin(2 * np.pi * t / span + 0.3 * i)[None]
    return rows


CASES = [(src, tm, noise) for src in ("small", "synthetic") for tm in (False, True) for noise in (False, True)]


@pytest.mark.parametrize("src,tm,noise", CASES)
def test_statics_match_dense_oracle(src, tm, noise):
    psrs = _small() if src == "small" else _synthetic()
    b = _batch(psrs, tm=tm, red=noise, ecorr=noise)
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    pc = b.plan()["curn"]
    rows = _rows(b, 5, seed=len(psrs))
    got = CO.lnl_of_statics(b, pc, rows)
    ref = CO.lnl_map(b, rows, X_GRID, G_GRID, K=6, models=_models(b) if tm else None)
    d = float(np.max(np.abs(got - ref)))
    print(f"\n[curn] {src} tm={tm} noise={noise}: max |d lnL| = {d:.1e} (|lnL| <= {np.max(np.abs(ref)):.1e})")
    assert d <= TOL
    # ldet is sum_a slogdet(I + A^2 phi~^1/2 Z_a phi~^1/2)
    from tests import os_oracle as OO
    Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    for g, gm in enumerate(G_GRID):
        sp = np.sqrt(OO.phi_tilde(6, gm, Tspan))
        Zh = pc["Z"] * sp[None, :, None] * sp[None, None, :]
        for k, xa in enumerate(X_GRID):
            ld = sum(np.linalg.slogdet(np.eye(12) + 10 ** (2 * xa) * Zh[a])[1] for a in range(b.n_psr))
            assert abs(pc["ldet"][g, k] - ld) <= 1e-9 * max(1.0, abs(ld))
    assert np.all(pc["eig"] >= 0) and pc["V"].shape == (b.n_psr, 3, 16, 16) and np.all(pc["V"][:, :, 12:] == 0)


def test_summaries_of_simple_maps():
    x = np.linspace(-16, -13, 31)
    gam = np.linspace(1, 6, 11)
    flat = CO.summaries(np.zeros((1, 11, 31)), x, gam)
    assert abs(flat["ln_bayes"][0]) < 1e-13                       # the prior is normalised on the grid
    np.testing.assert_allclose(flat["post_log10_A"][0], 1 / 3.0, rtol=1e-13)
    np.testing.assert_allclose(flat["post_gamma"][0], 1 / 5.0, rtol=1e-13)
    assert abs(flat["log10_A_ul"][0] - (-16 + 0.95 * 3)) < 1e-12
    assert flat["ml_gamma_index"][0] == 0 and flat["ml_log10_A_index"][0] == 0
    m = np.zeros((2, 11, 31))
    m[0, 4, 7] = m[0, 2, 9] = 1.0                                 # a tie: gamma-major, the lower index
    m[1, 10, 30] = 5.0
    s = CO.summaries(m, x, gam)
    assert (s["ml_gamma_index"][0], s["ml_log10_A_index"][0]) == (2, 9) and s["lnL_max"][0] == 1.0
    assert (s["ml_gamma_index"][1], s["ml_log10_A_index"][1]) == (10, 30)
    for r in range(2):
        assert abs(np.sum(CO.weights(x) * s["post_log10_A"][r]) - 1) < 1e-13
        assert abs(np.sum(CO.weights(gam) * s["post_gamma"][r]) - 1) < 1e-13
    u = CO.summaries(np.zeros((1, 1, 31)), x, [4.0], kind="uniform")
    assert -13.2 < u["log10_A_ul"][0] < -13.0                     # uniform in A: the mass sits at the top of the grid


def test_plan_weights_and_prior_match_oracle():
    b = _batch(_small())
    for kind in ("log-uniform", "uniform"):
        b.set_curn_likelihood(amplitude_prior=kind)
        pc = b.plan()["curn"]
        assert pc["V"].shape == (3, 57, 32, 32) and pc["ldet"].shape == (57, 97)
        np.testing.assert_allclose(pc["wg"], CO.weights(pc["gamma"]), rtol=1e-14)
        np.testing.assert_allclose(pc["wx"], CO.weights(pc["log10_A"]), rtol=1e-14)
        np.testing.assert_allclose(pc["prior"], CO.prior(pc["log10_A"], pc["gamma"], kind), rtol=1e-12)
    b.set_curn_likelihood(gamma=[13 / 3])
    assert np.array_equal(b.plan()["curn"]["wg"], [1.0])


def test_registration_leaves_other_statistics_unchanged():
    b = _batch(_small(), tm=True)
    b.set_optimal_statistic()
    b.set_fp_statistic(n_freqs=5)
    pl0 = b.plan()
    assert pl0["curn"] is None and b.curn_setup_s is None
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID)
    pl1 = b.plan()
    for sec in ("os", "fp"):
        for k, v in pl0[sec].items():
            if k != "setup_s":
                assert np.array_equal(np.asarray(v), np.asarray(pl1[sec][k])), (sec, k)
    assert pl1["curn"]["setup_s"] > 0 and b.curn_setup_s == pl1["curn"]["setup_s"]


@pytest.mark.parametrize("kw,match", [
    (dict(log10_A=[-15.0]), "log10_A needs 2..256"),
    (dict(log10_A=np.linspace(-18, -12, 257)), "log10_A needs 2..256"),
    (dict(gamma=np.linspace(0, 7, 257)), "gamma needs 1..256"),
    (dict(gamma=[]), "gamma needs 1..256"),
    (dict(log10_A=[-15.0, -15.0, -14.0]), "strictly increasing"),
    (dict(log10_A=[-14.0, -15.0]), "strictly increasing"),
    (dict(log10_A=[-15.0, np.nan]), "strictly increasing"),
    (dict(gamma=[1.0, np.inf]), "strictly increasing"),
    (dict(components=0), "components"),
    (dict(components=17), "components"),
    (dict(components=2.5), "components"),
    (dict(amplitude_prior="flat"), "amplitude_prior"),
    (dict(ul=0.0), "ul must be"),
    (dict(ul=1.0), "ul must be"),
    (dict(ul=np.nan), "ul must be"),
    (dict(Tspan=-1.0), "Tspan"),
])
def test_argument_checks(kw, match):
    b = _batch(_small())
    with pytest.raises(ValueError, match=match):
        b.set_curn_likelihood(**kw)


def test_missing_white_noise_raises_in_plan():
    b = _batch(_small(), white=False)
    b.set_curn_likelihood()
    with pytest.raises(ValueError, match="CURN likelihood needs white noise"):
        b.plan()


def test_curn_model_checks_refuse_before_any_launch():
    """``ptar_curn_reduce`` checks only the grid fields it reads, ``ptar_curn_grid`` those and the per-pulsar forms;
    both refuse a bad model before anything reaches a device."""
    import ctypes as C

    from pta_replicator_b200 import _cabi
    L = _cabi.lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)                                  # never read: every call below stops at its checks

    def model(**kw):
        f = dict(n_psr=1, nc=2, ncp=8, n_gamma=3, n_amp=6, V=p, lam=p, a2=p, ldet=p, log10_A=p, wg=p, wx=p, prior=p, ul=0.95)
        return _cabi.CurnModel(**{**f, **kw})

    calls = dict(reduce=lambda m: L.ptar_curn_reduce(p, 4, C.byref(m), *([p] * 7), None),
                 grid=lambda m: L.ptar_curn_grid(p, 4, C.byref(m), p, None))
    for kw, msg, which in ((dict(log10_A=None), "model arrays missing", calls), (dict(wg=None), "model arrays missing", calls),
                           (dict(wx=None), "model arrays missing", calls), (dict(prior=None), "model arrays missing", calls),
                           (dict(n_amp=1), "2 <= n_amp", calls), (dict(ul=1.0), "0 < ul < 1", calls),
                           (dict(V=None), "model arrays missing", ("grid",)), (dict(nc=0), "0 < nc <= 32", ("grid",))):
        for name in which:
            assert calls[name](model(**kw)) == -2, (name, kw)
            err = L.ptar_last_error().decode()
            assert msg in err and f"ptar_curn_{name}" in err, (name, kw, err)
