"""CPU tests of the anisotropy statics of the optimal statistic (``PulsarBatch.set_os_anisotropy``,
``plan()["os_aniso"]``): the plan's V and divisors applied in numpy against the dense oracle (tests/aniso_oracle.py,
a least-squares fit and two chi^2 minima, polarisation-tensor antenna patterns), the normalisations of both bases, the
argument and singularity checks and the registration's lifecycle.  ``plan_only`` batches: the 3 ``partim_small``
pulsars, the 4-pulsar synthetic case of test_optimal_statistic_cpu.py and an 8-pulsar synthetic case."""
import numpy as np
import pytest

from tests import aniso_oracle as AO
from tests import os_oracle as OO
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

K = 10
TOL = 1e-10


def _psrs(src):
    if src == "small":
        return _small()
    if src == "synthetic":
        return _synthetic()
    return _synthetic(seed=5, nep=(30, 35, 40, 45, 38, 42, 33, 50))


def _setup(src, tm, common, lmax, nside):
    b = _batch(_psrs(src), tm=tm)
    b.set_optimal_statistic(components=K, orfs=("hd",), log10_A_common=common)
    b.set_os_anisotropy(lmax=lmax, nside=nside)
    pl = b.plan()
    S0 = OO.statics(b, K=K, models=_models(b) if tm else None, templates=("hd",), log10_A_common=common)
    return b, pl["os"], pl["os_aniso"], S0


def _rows(b, R=6):
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    rows = np.random.default_rng(2).standard_normal((R, b.ld)) * 1e-6
    rows[:, ~live] = 0
    return rows


def _apply(pn, d):
    """The plan's statics applied to the pair correlations d [R, n_pairs]: the device's map columns."""
    return d @ pn["V"][:pn["n_col"], :pn["kd"]].T / pn["dsqrt"]


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


CASES = [("small", 0, 2), ("synthetic", 1, None), ("eight", 2, 1)]


@pytest.mark.parametrize("src,lmax,nside", CASES)
@pytest.mark.parametrize("tm", [False, True])
@pytest.mark.parametrize("common", [None, -14.5])
def test_plan_statics_match_dense_oracle(src, lmax, nside, tm, common):
    b, po, pn, S0 = _setup(src, tm, common, lmax, nside)
    pairs = S0["pairs"]
    d, t = AO.pair_correlations(b, S0, _rows(b))
    assert _rel(po["t_ab"], t) <= TOL
    got = _apply(pn, d)
    n_lm, n_z = pn["n_lm"], pn["n_z"]
    assert n_lm == (lmax + 1) ** 2 and n_z == n_lm - 1 and pn["kd"] == len(t)
    c, dchi2 = AO.sph_fit(d, t, AO.sph_templates(b, lmax, pairs))
    e_c, e_chi = _rel(got[:, :n_lm], c), 0.0
    assert e_c <= TOL
    if n_z:
        e_chi = _rel(np.sum(got[:, n_lm:n_lm + n_z] ** 2, axis=1), dchi2)
        assert e_chi <= TOL
    Tref = AO.sph_templates(b, lmax, pairs)
    assert _rel(pn["clm_cov"], np.linalg.inv((Tref * t) @ Tref.T)) <= TOL
    e_r = 0.0
    if nside is not None:
        from pta_replicator_b200.engine import healpix_ring_centres
        snr, sig = AO.radiometer(d, t, AO.radio_templates(b, healpix_ring_centres(nside), pairs))
        e_r = max(_rel(got[:, n_lm + n_z:], snr), _rel(pn["radio_sigma"], sig))
        assert e_r <= TOL and pn["n_sky"] == 12 * nside**2
    print(f"\n[os aniso] {src} lmax={lmax} nside={nside} tm={tm} common={common}: rel err c^ {e_c:.1e}, chi2 {e_chi:.1e}, "
          f"radiometer {e_r:.1e}")
    assert np.all(pn["V"][:, pn["kd"]:] == 0) and np.all(pn["V"][pn["n_col"]:] == 0)
    assert pn["V"].shape[0] % 64 == 0 and pn["kdp"] % 32 == 0


def test_lmax0_is_the_hd_amplitude():
    """c^_00 = sqrt(4 pi) A2[hd]: the l = 0 template is the HD template over sqrt(4 pi)."""
    b, po, pn, S0 = _setup("eight", True, None, 0, None)
    rows = _rows(b)
    d, t = AO.pair_correlations(b, S0, rows)
    a2 = OO.os_of_rows(b, S0, rows)["A2"][:, 0]
    assert _rel(_apply(pn, d)[:, 0], np.sqrt(4 * np.pi) * a2) <= TOL
    assert pn["n_z"] == 0 and pn["n_col"] == 1


def test_normalisations():
    """sqrt(4 pi) B_00 is the "hd" template of the optimal statistic on every pair; the radiometer's pixel sum tends to
    it as nside grows (pixelisation error only)."""
    b = _batch(_synthetic(seed=9, nep=(30,) * 12), tm=False)
    b.set_optimal_statistic(components=4, orfs=("hd",))
    b.set_os_anisotropy(lmax=0)
    pl = b.plan()
    hd = pl["os"]["orf"][0]
    e00 = float(np.max(np.abs(np.sqrt(4 * np.pi) * pl["os_aniso"]["T_sph"][0] - hd)))
    assert e00 <= 1e-15 * np.max(np.abs(hd))          # the two roundings of sqrt(4 pi) only
    errs = []
    for nside in (8, 16, 32):
        b.set_os_anisotropy(nside=nside)
        errs.append(float(np.max(np.abs(b.plan()["os_aniso"]["T_radio"].sum(axis=0) - hd))))
    print(f"\n[os aniso] sqrt(4 pi) B_00 - hd: {e00:.1e}; pixel sum - hd at nside 8, 16, 32: {np.array(errs)}")
    assert errs[2] < errs[1] < errs[0] < 5e-3 and errs[2] < 5e-4


def test_value_errors():
    b = _batch(_synthetic())
    with pytest.raises(ValueError, match="set_optimal_statistic"):
        b.set_os_anisotropy(lmax=2)
    b.set_optimal_statistic(components=K)
    with pytest.raises(ValueError, match="needs a basis"):
        b.set_os_anisotropy()
    for bad in (-1, 8, 2.0, True, "2"):
        with pytest.raises(ValueError, match="lmax"):
            b.set_os_anisotropy(lmax=bad)
    for bad in (0, 3, 64, 2.0, True):
        with pytest.raises(ValueError, match="nside"):
            b.set_os_anisotropy(nside=bad)
    for bad, msg in ((np.zeros((3, 3)), "shape"), (np.zeros((0, 2)), "empty"), (np.full((2, 2), np.nan), "finite"),
                     (np.zeros((12289, 2)), "at most")):
        with pytest.raises(ValueError, match=msg):
            b.set_os_anisotropy(sky=bad)
    with pytest.raises(ValueError, match="not both"):
        b.set_os_anisotropy(nside=2, sky=np.zeros((1, 2)) + 0.3)
    b.set_os_anisotropy(lmax=7)                        # the stated limit is accepted ...
    with pytest.raises(ValueError, match="singular"):  # ... and 64 coefficients on 6 pairs are rejected by the plan
        b.plan()
    b.set_os_anisotropy(lmax=1, sky=np.zeros((12288, 2)) + 0.3)
    small = _batch(_small())
    small.set_optimal_statistic(components=K)
    small.set_os_anisotropy(lmax=1)                    # 4 coefficients on 3 pairs
    with pytest.raises(ValueError, match="singular"):
        small.plan()
    # a radiometer pixel on the line of sight of one pulsar of a two-pulsar array: its pattern is 0, so F_kk = 0
    two = _batch(_synthetic(nep=(30, 40)))
    two.set_optimal_statistic(components=K, orfs=("hd",))
    u = AO.pulsar_units(two)[0]
    two.set_os_anisotropy(sky=[[np.arccos(u[2]), np.arctan2(u[1], u[0])]])
    with pytest.raises(ValueError, match="F_kk"):
        two.plan()


def test_registration_lifecycle():
    b = _batch(_synthetic())
    b.set_optimal_statistic(components=K)
    b.set_os_null("sky_scramble", n=4)
    b._compiled = object()
    b.set_os_anisotropy(lmax=1, nside=1)
    assert b._compiled is None
    pl = b.plan()
    assert pl["os_aniso"] is not None and b.os_aniso_setup_s >= 0 and pl["os_null"] is not None
    assert pl["os_aniso"]["n_col"] == 4 + 3 + 12
    d0 = pl["os_aniso"]["dsqrt"].copy()
    b.set_red(1, -12.5, 4.0, components=20)            # a recipe change re-derives the statics
    assert not np.allclose(d0, b.plan()["os_aniso"]["dsqrt"])
    b.set_optimal_statistic(components=K)              # clears the registration
    assert b.plan()["os_aniso"] is None
