"""CPU tests of the free spectrum's spectral refit (``pta_replicator_b200.spectra``, ``PulsarBatch.set_spectral_refit``,
``plan()["fs_refit"]``): the power law against the CURN prior bit for bit, the turnover against ``set_gwb``'s expression,
ldet against a direct sum over the free spectrum's eigenvalues, the eigen form on the plan's statics against the dense
refit oracle (tests/fs_refit_oracle.py) with a timing model, the independence of the registration and every argument
and plan-time check.  ``plan_only`` batches: the 3 ``partim_small`` pulsars and the 4-pulsar synthetic case of the
optimal-statistic tests."""
import numpy as np
import pytest

from pta_replicator_b200 import constants as const
from pta_replicator_b200 import spectra
from pta_replicator_b200.engine import _powerlaw_prior
from tests import fs_refit_oracle as RO
from tests.test_curn_likelihood_cpu import TOL, _rows
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic


def _user(rho2, x=(0.0, 1.0), y=(0.0,)):
    """A user model returning the fixed array ``rho2`` whatever f and Tspan."""
    return spectra.SpectralModel(np.asarray(x, float), np.asarray(y, float), lambda f, T, x, y: rho2)


def test_powerlaw_is_the_curn_prior_bit_for_bit():
    m = spectra.powerlaw()
    assert np.array_equal(m.x, np.linspace(-18, -12, 97)) and np.array_equal(m.y, np.linspace(0, 7, 57))
    T = 4.7e8
    f = np.arange(1, 15) / T
    r2 = m.rho2(f, T, m.x, m.y)
    assert r2.shape == (57, 97, 14)
    for iy, g in enumerate(m.y):
        ref = 10.0 ** (2 * m.x)[:, None] * _powerlaw_prior(f, g, T)[None, 0::2]
        assert np.array_equal(r2[iy], ref)


def test_turnover_is_set_gwbs_spectrum():
    rng = np.random.default_rng(5)
    T = 5.1e8
    f = np.arange(1, 31) / T
    worst = 0.0
    for _ in range(20):
        gamma, beta, power = rng.uniform(1, 6), rng.uniform(0.5, 2), rng.uniform(0.5, 3)
        x, y = np.sort(rng.uniform(-16, -13, 3)), np.sort(rng.uniform(-9.5, -7.5, 2))
        r2 = spectra.turnover(x, y, gamma, beta, power).rho2(f, T, x, y)
        alpha = -0.5 * (gamma - 3)
        for iy, lf0 in enumerate(y):
            for ix, la in enumerate(x):
                hcf = 10**la * (f / const.GWB_F1YR) ** alpha                          # set_gwb's expression
                hcf = hcf / (1 + (f / 10**lf0) ** (power * (alpha - beta))) ** (1 / power)
                ref = hcf**2 / (12 * np.pi**2 * f**3 * T)
                worst = max(worst, float(np.max(np.abs(r2[iy, ix] - ref) / ref)))
    assert worst <= 1e-14
    # f0 far below f_1: set_gwb's power law (turnover=False)
    x = np.array([-15.0, -14.0])
    r2 = spectra.turnover(x, [-14.0], 13 / 3).rho2(f, T, x, np.array([-14.0]))
    pl = (10.0 ** x[:, None] * (f / const.GWB_F1YR) ** (-2 / 3)) ** 2 / (12 * np.pi**2 * f**3 * T)
    np.testing.assert_allclose(r2[0], pl, rtol=1e-8)
    # ... which is spectra.powerlaw up to the year of set_gwb (1 / 3.16e7 s against 365.25 d)
    ratio = r2[0] / spectra.powerlaw(x, [13 / 3]).rho2(f, T, x, np.array([13 / 3]))[0]
    np.testing.assert_allclose(ratio, (const.YEAR_IN_SEC * const.GWB_F1YR) ** (4 / 3), rtol=1e-8)


@pytest.mark.parametrize("orf", [None, "hd"])
def test_ldet_is_the_direct_sum_over_the_eigenvalues(orf):
    b = _batch(_synthetic(), tm=True)
    K = 5
    b.set_free_spectrum(components=K, orf=orf)
    m = spectra.powerlaw(np.linspace(-16, -13, 7), [2.0, 13 / 3, 5.5])
    b.set_spectral_refit({"pl": m, "to": spectra.turnover(np.linspace(-16, -13, 4), [-9.0, -8.5])})
    pl = b.plan()
    pf, pr = pl["fs"], pl["fs_refit"]
    assert pr["setup_s"] > 0 and b.fs_refit_setup_s == pr["setup_s"]
    for name in ("pl", "to"):
        pm = pr["models"][name]
        Ny, Nx = len(pm["y"]), len(pm["x"])
        assert pm["rho2"].shape == (Ny, Nx, K) and np.array_equal(pm["rho2_kt"], pm["rho2"].reshape(-1, K).T)
        for prefix, lam in (("", pf["eig"].transpose(1, 0, 2).reshape(K, -1)),) + ((("hd_", pf["hd_eig"]),) if orf else ()):
            ref = np.log1p(pm["rho2"][..., None] * lam[None, None]).sum(axis=(2, 3))
            assert pm[prefix + "ldet"].shape == (Ny, Nx)
            np.testing.assert_allclose(pm[prefix + "ldet"], ref, rtol=1e-13)
        assert ("hd_ldet" in pm) == (orf is not None)
        np.testing.assert_allclose((pm["wg"].sum() * (pm["wx"] @ pm["prior"])), 1.0, rtol=1e-14)


@pytest.mark.parametrize("src,tm,orf,K", [("small", True, "hd", 4), ("synthetic", True, "dipole", 3),
                                          ("synthetic", False, None, 1)])
def test_eigen_form_matches_dense_refit_oracle(src, tm, orf, K):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    b.set_free_spectrum(components=K, orf=orf)
    x, g = np.linspace(-15.0, -13.5, 3), np.array([2.0, 13 / 3])
    b.set_spectral_refit({"pl": spectra.powerlaw(x, g), "to": spectra.turnover(x, [-8.8, -8.2])})
    pl = b.plan()
    pf, pr = pl["fs"], pl["fs_refit"]
    rows = _rows(b, 4, seed=K)
    models = _models(b) if tm else None
    for name in ("pl", "to"):
        pm = pr["models"][name]
        for prefix, o in (("", None),) + ((("hd_", orf),) if orf else ()):
            got = RO.lnl_of_statics(b, pf, pm, rows, prefix)
            ref = RO.lnl_map(b, rows, pm["rho2"].reshape(-1, K), orf=o, models=models).reshape(got.shape)
            d = float(np.max(np.abs(got - ref)))
            print(f"\n[fs refit] {src} tm={tm} K={K} {name} {prefix or 'uncorrelated'}: max |d lnL| = {d:.1e}")
            assert d <= TOL


def test_registration_leaves_every_other_plan_unchanged():
    b = _batch(_small(), tm=True)
    assert b.fs_refit_setup_s is None
    b.set_optimal_statistic()
    b.set_curn_likelihood(log10_A=np.linspace(-15.5, -13, 4), gamma=[2.0, 4.0])
    b.set_hd_likelihood()
    b.set_free_spectrum(components=5, orf="hd")
    pl0 = b.plan()
    assert pl0["fs_refit"] is None
    b.set_spectral_refit({"pl": spectra.powerlaw(np.linspace(-16, -13, 5), [3.0, 4.0])})
    pl1 = b.plan()
    for sec in ("os", "curn", "hd", "fs"):
        assert pl0[sec].keys() == pl1[sec].keys()
        for k, v in pl0[sec].items():
            if k != "setup_s":
                assert np.array_equal(np.asarray(v), np.asarray(pl1[sec][k])), (sec, k)
    # the statics follow the free spectrum as it stands at plan()
    b.set_free_spectrum(components=3)
    pr = b.plan()["fs_refit"]
    assert pr["models"]["pl"]["rho2"].shape == (2, 5, 3) and "hd_ldet" not in pr["models"]["pl"]


def test_refit_needs_a_free_spectrum_without_a_common_process():
    b = _batch(_small())
    with pytest.raises(ValueError, match="no free-spectrum likelihood registered"):
        b.set_spectral_refit({"pl": spectra.powerlaw()})
    b.set_free_spectrum(components=4, log10_A_common=-14.5)
    b.set_spectral_refit({"pl": spectra.powerlaw()})
    with pytest.raises(ValueError, match="without log10_A_common.*count those bins twice"):
        b.plan()


K4 = np.ones((1, 2, 4))


@pytest.mark.parametrize("models,kw,match", [
    ({}, {}, "non-empty dict"),
    ([("pl", None)], {}, "non-empty dict"),
    ({"1pl": spectra.powerlaw()}, {}, "bad refit model name"),
    ({"p-l": spectra.powerlaw()}, {}, "bad refit model name"),
    ({"": spectra.powerlaw()}, {}, "bad refit model name"),
    ({"pl": (np.zeros(2), np.zeros(1), None)}, {}, "SpectralModel"),
    ({"pl": spectra.powerlaw([-14.0])}, {}, "x of refit model 'pl' needs 2..256"),
    ({"pl": spectra.powerlaw(np.linspace(-18, -12, 257))}, {}, "x of refit model 'pl' needs 2..256"),
    ({"pl": spectra.powerlaw([-14.0, -15.0])}, {}, "strictly increasing"),
    ({"pl": spectra.powerlaw(gamma=[])}, {}, "y of refit model 'pl' needs 1..256"),
    ({"pl": spectra.powerlaw(gamma=[1.0, np.nan])}, {}, "strictly increasing"),
    ({"pl": spectra.powerlaw()}, dict(amplitude_prior="flat"), "amplitude_prior"),
    ({"pl": spectra.powerlaw()}, dict(ul=1.0), "ul must be"),
    ({"pl": spectra.powerlaw()}, dict(ul=0.0), "ul must be"),
    ({"u": _user(np.ones((1, 2, 3)))}, {}, r"rho2 of refit model 'u' has shape \(1, 2, 3\), expected .* \(1, 2, 4\)"),
    ({"u": _user(np.where(np.arange(8).reshape(1, 2, 4) == 6, np.nan, K4))}, {},
     r"rho2 of refit model 'u' is nan at x = 1.0, y = 0.0 \(grid point \(0, 1\)\) in bin 3"),
    ({"u": _user(np.where(np.arange(8).reshape(1, 2, 4) == 1, -1.0, K4))}, {},
     r"rho2 of refit model 'u' is -1.0 at x = 0.0, y = 0.0 \(grid point \(0, 0\)\) in bin 2"),
    ({"u": _user(np.where(np.arange(8).reshape(1, 2, 4) == 3, np.inf, K4))}, {}, r"is inf .* in bin 4"),
])
def test_argument_checks(models, kw, match):
    b = _batch(_small())
    b.set_free_spectrum(components=4)
    with pytest.raises(ValueError, match=match):
        b.set_spectral_refit(models, **kw)
    assert b._fs_refit is None


def test_turnover_argument_checks():
    with pytest.raises(ValueError, match="gamma must be finite"):
        spectra.turnover(gamma=np.nan)
    with pytest.raises(ValueError, match="power must be positive"):
        spectra.turnover(power=0.0)
