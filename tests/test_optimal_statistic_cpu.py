"""CPU tests of the optimal statistic's host statics (``PulsarBatch.set_optimal_statistic``, ``plan()["os"]``) against
the dense oracle (tests/os_oracle.py), and of the argument checks.  ``plan_only`` batches: the 3 ``partim_small``
pulsars and a synthetic case with several backends and 1-s ECORR."""
import os

import numpy as np
import pytest

from tests import os_oracle as OO
from tests import timing_oracle as TO
from tests.fixtures import GOLD

# Woodbury (host statics) and the dense null-space solve (oracle) round differently.  Measured worst relative
# differences on these cases: 2.9e-13 (C), 2.2e-14 (Z), 8.5e-14 (t), 1.2e-13 (F^-1); the bound leaves room for
# other BLAS builds and worse-conditioned recipes.
TOL = 1e-10


def _small():
    from pta_replicator_b200 import load_from_directories, make_ideal
    psrs = load_from_directories(os.path.join(GOLD, "partim_small", "par"), os.path.join(GOLD, "partim_small", "tim"))
    for p in psrs:
        make_ideal(p)
    return psrs


def _synthetic(seed=3, nep=(40, 55, 70, 48)):
    """4 pulsars, epochs of 3-6 sub-band TOAs within 1 s, 3 backends cycling per epoch (flag f)."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, ne in enumerate(nep):
        ep = np.sort(rng.uniform(53000.0, 58800.0, ne))
        nsub = rng.integers(3, 7, ne)
        mjd = np.concatenate([e + rng.uniform(0, 0.9, k) / 86400.0 for e, k in zip(ep, nsub)])
        be = np.concatenate([[("A", "B", "C")[q % 3]] * k for q, k in enumerate(nsub)])
        err = rng.uniform(0.2, 2.0, mjd.size)
        p = pulsar_from_arrays(f"S{j}", {"RAJ": float(rng.uniform(0, 24)), "DECJ": float(rng.uniform(-60, 60))},
                               mjd.astype(np.longdouble), err, flags=[{"f": f} for f in be])
        make_ideal(p)
        out.append(p)
    return out


def _batch(psrs, red=True, ecorr=True, tm=False, white=True):
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs, plan_only=True)
    for i in range(b.n_psr):
        if white:
            b.set_white(i, efac=1.1, log10_equad=-6.5)
        if ecorr:
            b.set_ecorr(i, -6.3, coarsegrain=1.0 / 86400.0)
        if red:
            b.set_red(i, -13.8 - 0.1 * i, 3.5 + 0.3 * i, components=20)
        if tm:
            b.set_timing_model(i, poly=2, jumps="f")
    return b


def _models(b):
    """Oracle design matrices (its own construction) in engine order."""
    out = []
    for i, p in enumerate(b.psrs):
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        fv = [f.get("f") for f in p.toas.table["flags"]]
        out.append(TO.timing_design_matrix(t, 2, fv)[b.order[i]])
    return out


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / np.max(np.abs(b)))


CASES = [(src, tm, common) for src in ("small", "synthetic") for tm in (False, True) for common in (None, -14.5)]


@pytest.mark.parametrize("src,tm,common", CASES)
def test_statics_match_dense_oracle(src, tm, common):
    psrs = _small() if src == "small" else _synthetic()
    b = _batch(psrs, tm=tm)
    orfs = ("hd", "monopole", "dipole") if b.n_psr > 3 else ("hd", "monopole")
    b.set_optimal_statistic(components=10, orfs=orfs, log10_A_common=common)
    po = b.plan()["os"]
    S = OO.statics(b, K=10, log10_A_common=common, models=_models(b) if tm else None, templates=orfs)
    worst = {}
    worst["C"] = max(_rel(po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :20], S["C"][i]) for i in range(b.n_psr))
    worst["Z"] = max(_rel(po["Z"][i], S["Z"][i]) for i in range(b.n_psr))
    worst["t"] = _rel(po["t"], S["t"])
    worst["W"] = _rel(po["orf"], S["W"])
    worst["Finv"] = _rel(po["finv"], S["Finv"])
    print(f"\n[os statics] {src} tm={tm} common={common}: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert max(worst.values()) < TOL, worst
    assert np.all(po["C"][:, 20:] == 0)
    # alignment slots of the packed axis carry no weight
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    assert np.all(po["C"][~live] == 0)
    # the statistic of some rows from the plan's statics equals the oracle's
    rows = np.random.default_rng(1).standard_normal((3, b.ld)) * 1e-6
    rows[:, ~live] = 0
    ref = OO.os_of_rows(b, S, rows)
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :20]
                  for i in range(b.n_psr)], axis=1) * np.sqrt(po["phi"])
    d = np.einsum("rpj,rpj->rp", X[:, pa], X[:, pb])
    assert np.max(np.abs(d / po["t_ab"] - ref["rho"]) / po["sigma"]) < 1e-8
    assert np.max(np.abs(d @ po["orf"].T / po["dsqrt"] - ref["snr"])) < 1e-8


@pytest.mark.parametrize("src", ["small", "synthetic"])
def test_c_annihilates_the_timing_model(src):
    b = _batch(_small() if src == "small" else _synthetic(), tm=True)
    b.set_optimal_statistic(components=14, orfs=("hd",))
    po = b.plan()["os"]
    M = _models(b)
    worst = 0.0
    for i in range(b.n_psr):
        Ca = po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :28]
        worst = max(worst, float(np.max(np.abs(Ca.T @ M[i])) / (np.linalg.norm(Ca) * np.linalg.norm(M[i]))))
    print(f"\n[os statics] {src}: max |C^T M| / (|C| |M|) = {worst:.1e}")
    assert worst < 1e-10


def test_hd_template_and_null_sigmas():
    b = _batch(_synthetic())
    b.set_optimal_statistic(orfs=("hd", "dipole", np.eye(4) + 0.25))
    po = b.plan()["os"]
    h, c = OO.hd_closed_form(b)
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    assert np.allclose(po["orf"][0], h[pa, pb], rtol=0, atol=1e-13)
    assert np.allclose(po["orf"][1], c[pa, pb], rtol=0, atol=1e-13)
    assert np.all(po["orf"][2] == 0.25)
    assert np.allclose(po["sigma"], po["t_ab"] ** -0.5)
    assert np.allclose(po["A2_sigma"], 1 / np.sqrt((po["orf"] ** 2) @ po["t_ab"]))
    assert np.allclose(po["finv"] @ po["F"], np.eye(3), atol=1e-9)
    assert po["names"] == ["hd", "dipole", "matrix"]
    assert b.os_setup_s is not None and b.os_setup_s >= 0


def test_recipe_changes_after_registration_change_the_statics():
    b = _batch(_synthetic())
    b.set_optimal_statistic(orfs=("hd",))
    t0 = b.plan()["os"]["t_ab"].copy()
    b._compiled = object()
    b.set_red(1, -12.5, 4.0, components=20)
    assert b._compiled is None
    t1 = b.plan()["os"]["t_ab"].copy()
    assert not np.allclose(t0, t1)
    b._compiled = object()
    b.set_timing_model(2, poly=2)
    assert b._compiled is None
    t2 = b.plan()["os"]["t_ab"]
    assert not np.allclose(t1, t2)
    b.set_white(0, efac=2.0)
    assert not np.allclose(t2, b.plan()["os"]["t_ab"])


def test_value_errors():
    from pta_replicator_b200.engine import PulsarBatch
    psrs = _synthetic()
    b = _batch(psrs)
    for bad in (0, 17, 2.5):
        with pytest.raises(ValueError, match="components"):
            b.set_optimal_statistic(components=bad)
    with pytest.raises(ValueError, match="templates"):
        b.set_optimal_statistic(orfs=("hd", "monopole", "dipole", "hd", "monopole"))
    with pytest.raises(ValueError, match="templates"):
        b.set_optimal_statistic(orfs=())
    with pytest.raises(ValueError, match="unknown ORF template"):
        b.set_optimal_statistic(orfs=("quadrupole",))
    with pytest.raises(ValueError, match="must be \\[4, 4\\]"):
        b.set_optimal_statistic(orfs=(np.eye(3),))
    asym = np.eye(4)
    asym[0, 1] = 0.3
    with pytest.raises(ValueError, match="symmetric"):
        b.set_optimal_statistic(orfs=(asym,))
    with pytest.raises(ValueError, match="finite"):
        b.set_optimal_statistic(orfs=(np.full((4, 4), np.nan),))
    with pytest.raises(ValueError, match="at least 2 pulsars"):
        PulsarBatch(psrs[:1], plan_only=True).set_optimal_statistic()
    big = PulsarBatch(psrs, plan_only=True)
    big.n_psr = 257                      # the pair kernel's limit is stated as 256 pulsars
    with pytest.raises(ValueError, match="at most 256 pulsars"):
        big.set_optimal_statistic()
    # singular F: two identical templates
    b.set_optimal_statistic(orfs=("hd", "hd"))
    with pytest.raises(ValueError, match="singular"):
        b.plan()
    # a pulsar without white noise
    nw = _batch(psrs, white=False)
    nw.set_white(0, efac=1.0)
    nw.set_optimal_statistic()
    with pytest.raises(ValueError, match="set_white"):
        nw.plan()
    # zero white variance on some TOAs (efac 0 for one backend, no equad): P is not positive definite
    zw = _batch(psrs)
    zw.set_white(2, efac=np.array([1.0, 0.0, 1.0]), log10_equad=np.array([-np.inf, -np.inf, -np.inf]), flagid="f",
                 flags=["A", "B", "C"])
    zw.set_optimal_statistic()
    with pytest.raises(ValueError, match="zero white-noise variance"):
        zw.plan()
