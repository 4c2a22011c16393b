"""CPU tests of the factorised free-spectrum likelihood's host statics (``PulsarBatch.set_free_spectrum``,
``plan()["fs"]``): against the dense oracle (tests/fs_oracle.py) with and without a timing model, ECORR, red noise and
the conditioning common process; the conditioning against a direct Woodbury with the common process on the other bins;
the tie of every bin to the one-component CURN and HD likelihoods at Tspan / k; the independence of the registration
and the argument checks.  ``plan_only`` batches: the 3 ``partim_small`` pulsars and the 4-pulsar synthetic case of the
optimal-statistic tests."""
import numpy as np
import pytest

from pta_replicator_b200.engine import _powerlaw_prior, _sincos_basis
from tests import fs_oracle as FO
from tests.test_curn_likelihood_cpu import TOL, _rows
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

R_GRID = np.linspace(-8.5, -5.5, 5)

# (source, timing model, ECORR and red noise, log10_A_common, ORF, K)
CASES = [("small", False, True, None, None, 5), ("small", True, True, None, "hd", 5),
         ("small", True, False, -13.5, "hd", 4), ("synthetic", False, True, -14.0, None, 6),
         ("synthetic", True, True, -14.0, "dipole", 3), ("synthetic", True, False, None, "monopole", 1)]


def _psrs(src):
    return _small() if src == "small" else _synthetic()


@pytest.mark.parametrize("src,tm,noise,common,orf,K", CASES)
def test_statics_match_dense_oracle(src, tm, noise, common, orf, K):
    b = _batch(_psrs(src), tm=tm, red=noise, ecorr=noise)
    b.set_free_spectrum(log10_rho=R_GRID, components=K, orf=orf, log10_A_common=common)
    pf = b.plan()["fs"]
    models = _models(b) if tm else None
    rows = _rows(b, 4, seed=K)
    kw = dict(models=models, log10_A_common=common)
    Z = FO.z_blocks(b, K, **kw)
    assert np.max(np.abs(pf["Z"] - Z)) <= 1e-10 * np.max(np.abs(Z))
    lam = np.linalg.eigvalsh(Z)
    assert np.all(np.abs(pf["eig"] - lam) <= 1e-10 * np.max(lam, axis=2, keepdims=True))
    ldet = np.log1p(pf["a2"][None, None, :, None] * lam[:, :, None, :]).sum(axis=(0, 3))
    assert np.all(np.abs(pf["ldet"] - ldet) <= 1e-9 * np.maximum(1.0, np.abs(ldet)))
    ref = FO.lnl_map(b, rows, R_GRID, K, **kw)
    d = float(np.max(np.abs(FO.lnl_of_statics(b, pf, rows) - ref)))
    print(f"\n[fs] {src} tm={tm} noise={noise} common={common} K={K}: max |d lnL| = {d:.1e}")
    assert d <= TOL
    n, n2p, npad = 2 * b.n_psr, pf["n2p"], pf["np"]
    assert pf["V"].shape == (K, npad, n2p) and np.all(pf["V"][:, n:] == 0) and np.all(pf["V"][:, :, n:] == 0)
    assert pf["lam"].shape == (K, npad) and np.all(pf["lam"][:, n:] == 0) and np.all(pf["eig"] >= 0)
    if orf is not None:
        ref = FO.lnl_map(b, rows, R_GRID, K, orf=orf, **kw)
        d = float(np.max(np.abs(FO.lnl_of_statics(b, pf, rows, "hd_") - ref)))
        print(f"[fs] correlated model ({orf}): max |d lnL| = {d:.1e}")
        assert d <= TOL and pf["hd_V"].shape == (K, npad, n2p) and np.all(pf["hd_V"][:, n:] == 0)


@pytest.mark.parametrize("tm", [False, True])
def test_conditioning_equals_direct_woodbury(tm):
    """C_a,k and Z_a[k] of the rank update on the basis against _pinv_apply with the common process on F_-k."""
    b = _batch(_synthetic(), tm=tm)
    K, common = 5, -13.8
    b.set_free_spectrum(log10_rho=R_GRID, components=K, log10_A_common=common)
    pf = b.plan()["fs"]
    T = b._fs["Tspan"]
    f = np.arange(1, K + 1) / T
    phi = 10.0 ** (2 * common) * _powerlaw_prior(f, 13 / 3, T)
    dvar = b._white_variances("test")
    for k in range(K):
        rest = np.r_[0:2 * k, 2 * k + 2:2 * K]
        for a in range(b.n_psr):
            s, n = b.toa_off[a], b.ntoa[a]
            F = _sincos_basis(b.t_tdb[a], f)
            Ca = b._pinv_apply(a, dvar[a], F[:, 2 * k:2 * k + 2], (F[:, rest], phi[rest]))
            got = pf["C"][s:s + n, 2 * k:2 * k + 2]
            assert np.max(np.abs(got - Ca)) <= 1e-10 * np.max(np.abs(Ca))
            Za = F[:, 2 * k:2 * k + 2].T @ Ca
            assert np.max(np.abs(pf["Z"][a, k] - 0.5 * (Za + Za.T))) <= 1e-10 * np.max(np.abs(Za))


@pytest.mark.parametrize("tm", [False, True])
def test_bins_tie_to_one_component_curn_and_hd(tm):
    """Bin k is the CURN / HD likelihood of components=1 at Tspan / k: its eigenvalues times phi~ are theirs."""
    b = _batch(_small(), tm=tm)
    K, g = 4, 3.0
    b.set_free_spectrum(log10_rho=R_GRID, components=K, orf="hd")
    pf = b.plan()["fs"]
    T = b._fs["Tspan"]
    for k in range(1, K + 1):
        b.set_curn_likelihood(log10_A=[-15.0, -14.0], gamma=[g], components=1, Tspan=T / k)
        b.set_hd_likelihood("hd")
        pl = b.plan()
        pt = _powerlaw_prior([k / T], g, T / k)[0]
        lc = pl["curn"]["eig"][:, 0, :]                                    # [P, 2]
        np.testing.assert_allclose(pf["eig"][:, k - 1] * pt, lc, rtol=1e-10, atol=1e-12 * lc.max())
        lh = pl["hd"]["eig"][0]
        np.testing.assert_allclose(pf["hd_eig"][k - 1] * pt, lh, rtol=1e-10, atol=1e-12 * lh.max())


def test_identity_orf_reproduces_uncorrelated_model():
    b = _batch(_synthetic(), tm=True)
    b.set_free_spectrum(log10_rho=R_GRID, components=4, orf=np.eye(b.n_psr))
    pf = b.plan()["fs"]
    np.testing.assert_allclose(pf["hd_eig"], np.sort(pf["eig"].transpose(1, 0, 2).reshape(4, -1), axis=1), rtol=1e-11)
    np.testing.assert_allclose(pf["hd_ldet"], pf["ldet"], rtol=1e-12)
    rows = _rows(b, 3, seed=5)
    np.testing.assert_allclose(FO.lnl_of_statics(b, pf, rows, "hd_"), FO.lnl_of_statics(b, pf, rows), rtol=0, atol=1e-9)


def test_registration_leaves_other_statistics_unchanged():
    b = _batch(_small(), tm=True)
    for key in ("os", "os_null", "os_aniso", "os_pf", "fp", "fe", "curn", "hd", "rn", "bwm", "fs"):
        assert getattr(b, f"{key}_setup_s") is None, key               # a fresh batch has spent no time on any statics
    b.set_optimal_statistic()
    b.set_fp_statistic(n_freqs=5)
    b.set_curn_likelihood(log10_A=np.linspace(-15.5, -13, 4), gamma=[2.0, 4.0])
    b.set_hd_likelihood()
    b.set_red_noise_likelihood(log10_A=np.linspace(-15.5, -13, 4), gamma=[3.0], components=5)
    pl0 = b.plan()
    assert pl0["fs"] is None
    b.set_free_spectrum(orf="hd", log10_A_common=-14.0)
    pl1 = b.plan()
    for sec in ("os", "fp", "curn", "hd", "rn"):
        for k, v in pl0[sec].items():
            if k != "setup_s":
                assert np.array_equal(np.asarray(v), np.asarray(pl1[sec][k])), (sec, k)
    assert pl1["fs"]["setup_s"] > 0 and b.fs_setup_s == pl1["fs"]["setup_s"]


def test_default_grid_and_outputs():
    b = _batch(_synthetic())
    b.set_free_spectrum()
    pf = b.plan()["fs"]
    assert np.array_equal(pf["log10_A"], np.linspace(-10, -4, 121)) and pf["nc"] == 28 and pf["ncp"] == 32
    np.testing.assert_allclose(pf["freqs"], np.arange(1, 15) / b._fs["Tspan"], rtol=1e-15)
    assert "hd_V" not in pf and np.array_equal(pf["wg"], [1.0])
    np.testing.assert_allclose(pf["wx"] @ pf["prior"], 1.0, rtol=1e-14)


@pytest.mark.parametrize("kw,match", [
    (dict(log10_rho=[-7.0]), "log10_rho needs 2..256"),
    (dict(log10_rho=np.linspace(-10, -4, 257)), "log10_rho needs 2..256"),
    (dict(log10_rho=[-7.0, -8.0]), "strictly increasing"),
    (dict(log10_rho=[-7.0, np.nan]), "strictly increasing"),
    (dict(components=0), "components"),
    (dict(components=33), "components"),
    (dict(rho_prior="flat"), "amplitude_prior"),
    (dict(ul=1.0), "ul must be"),
    (dict(Tspan=0.0), "Tspan"),
    (dict(orf="quadrupole"), "unknown ORF template"),
    (dict(orf=np.eye(2)), "must be \\[3, 3\\]"),
    (dict(orf=-np.eye(3)), "not positive semi-definite"),
    (dict(log10_A_common=np.inf), "log10_A_common"),
    (dict(gamma_common=np.nan), "gamma_common"),
])
def test_argument_checks(kw, match):
    b = _batch(_small())
    with pytest.raises(ValueError, match=match):
        b.set_free_spectrum(**kw)


def test_orf_needs_two_pulsars():
    b = _batch(_small()[:1])
    b.set_free_spectrum(components=3)                  # the uncorrelated model works on one pulsar
    assert b.plan()["fs"]["V"].shape == (3, 32, 8)
    with pytest.raises(ValueError, match="at least 2 pulsars"):
        b.set_free_spectrum(orf="hd")


def test_missing_white_noise_raises_in_plan():
    b = _batch(_small(), white=False)
    b.set_free_spectrum()
    with pytest.raises(ValueError, match="free-spectrum likelihood needs white noise"):
        b.plan()
