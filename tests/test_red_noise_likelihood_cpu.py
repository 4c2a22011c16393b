"""CPU tests of the single-pulsar red-noise likelihood's host statics (``PulsarBatch.set_red_noise_likelihood``,
``plan()["rn"]``) against the dense oracle (tests/rn_oracle.py), of its basis and noise model, of the plan-time errors and
of the argument checks.  ``plan_only`` batches: the 3 ``partim_small`` pulsars (122 TOAs each), the 4-pulsar synthetic
case of the optimal-statistic tests and a one-pulsar batch, with and without a timing model and a common process; the
recipes carry red noise (20 components) that the statistic must leave out."""
import numpy as np
import pytest

from tests import rn_oracle as RO
from tests.test_curn_likelihood_cpu import G_GRID, TOL, X_GRID, _rows
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# (source, timing model, log10_A_common, K, gamma grid)
CASES = [("small", False, None, 14, G_GRID), ("small", True, None, 30, G_GRID), ("synthetic", True, -14.5, 14, G_GRID),
         ("synthetic", False, -14.5, 1, G_GRID), ("small", True, -14.0, 30, np.array([13 / 3])),
         ("one", True, None, 14, G_GRID), ("one", False, -14.5, 30, np.array([3.0]))]


def _psrs(src):
    return _small() if src == "small" else _synthetic() if src == "synthetic" else _small()[:1]


@pytest.mark.parametrize("src,tm,common,K,gam", CASES)
def test_statics_match_dense_oracle(src, tm, common, K, gam):
    b = _batch(_psrs(src), tm=tm)
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=gam, components=K, log10_A_common=common)
    pr = b.plan()["rn"]
    rows = _rows(b, 5, seed=b.n_psr + K)
    models = _models(b) if tm else None
    got = RO.lnl_of_statics(b, pr, rows)
    ref = RO.lnl_map(b, rows, X_GRID, gam, K=K, models=models, log10_A_common=common)
    d = float(np.max(np.abs(got - ref)))
    print(f"\n[rn] {src} tm={tm} common={common} K={K} Ng={len(gam)}: max |d lnL| = {d:.1e} "
          f"(|lnL| <= {np.max(np.abs(ref)):.1e})")
    assert d <= TOL
    ld = RO.ldet(b, X_GRID, gam, K=K, models=models, log10_A_common=common)
    assert np.all(np.abs(pr["ldet"] - ld) <= 1e-9 * np.maximum(1.0, np.abs(ld)))
    P, nc, ncp = b.n_psr, 2 * K, (2 * K + 7) // 8 * 8
    assert pr["V"].shape == (P, len(gam), ncp, ncp) and np.all(pr["V"][:, :, nc:] == 0) and np.all(pr["V"][..., nc:] == 0)
    assert pr["ldet"].shape == (P, len(gam), len(X_GRID)) and np.all(pr["eig"] >= 0) and pr["eig"].shape == (P, len(gam), nc)


def test_own_red_noise_is_left_out_but_still_enters_curn():
    kw = dict(log10_A=X_GRID, gamma=G_GRID, components=6)
    red, white = _batch(_small(), red=True, tm=True), _batch(_small(), red=False, tm=True)
    for b in (red, white):
        b.set_red_noise_likelihood(**kw)
        b.set_curn_likelihood(**kw)
    pr, pw = red.plan(), white.plan()
    for k in ("C", "Z", "V", "eig", "ldet"):
        assert np.array_equal(pr["rn"][k], pw["rn"][k]), k        # the recipe's red noise never enters the statics
    assert not np.allclose(pr["curn"]["Z"], pw["curn"]["Z"], rtol=1e-3)   # while the CURN noise model holds it


def test_default_basis_is_set_red_basis():
    b = _batch(_synthetic(), red=False)
    for i in range(b.n_psr):
        b.set_red(i, -14.0, 3.0)                                       # set_red's default: 30 components on T_a
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID)
    pr = b.plan()["rn"]
    assert np.array_equal(pr["freqs"], np.stack(b._red["f"]))
    assert np.array_equal(pr["Tspan"], [t.max() - t.min() for t in b.t_tdb])
    assert len({float(T) for T in pr["Tspan"]}) == b.n_psr               # each pulsar on its own span
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=4, Tspan=3e8)
    pr = b.plan()["rn"]
    assert np.array_equal(pr["freqs"], np.tile(np.arange(1, 5) / 3e8, (b.n_psr, 1)))
    assert np.array_equal(pr["Tspan"], [3e8] * b.n_psr)


def test_plan_weights_and_prior_match_curn():
    b = _batch(_small())
    for kind in ("log-uniform", "uniform"):
        b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=3, amplitude_prior=kind, ul=0.9)
        b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=3, amplitude_prior=kind, ul=0.9)
        pl = b.plan()
        for k in ("wg", "wx", "prior", "a2", "log10_A", "gamma", "ul"):
            assert np.array_equal(pl["rn"][k], pl["curn"][k]), k


def test_registration_leaves_other_statistics_unchanged():
    b = _batch(_small(), tm=True)
    b.set_optimal_statistic()
    b.set_fp_statistic(n_freqs=5)
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    b.set_hd_likelihood()
    pl0 = b.plan()
    assert pl0["rn"] is None and b.rn_setup_s is None
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID)
    pl1 = b.plan()
    for sec in ("os", "fp", "curn", "hd"):
        for k, v in pl0[sec].items():
            if k != "setup_s":
                assert np.array_equal(np.asarray(v), np.asarray(pl1[sec][k])), (sec, k)
    assert pl1["rn"]["setup_s"] > 0 and b.rn_setup_s == pl1["rn"]["setup_s"]


@pytest.mark.parametrize("kw,match", [
    (dict(log10_A=[-15.0]), "log10_A needs 2..256"),
    (dict(gamma=np.linspace(0, 7, 257)), "gamma needs 1..256"),
    (dict(log10_A=[-14.0, -15.0]), "strictly increasing"),
    (dict(gamma=[1.0, np.nan]), "strictly increasing"),
    (dict(components=0), "components"),
    (dict(components=33), "components"),
    (dict(components=True), "components"),
    (dict(amplitude_prior="flat"), "amplitude_prior"),
    (dict(ul=1.0), "ul must be"),
    (dict(ul=-0.5), "ul must be"),
    (dict(Tspan=0.0), "Tspan"),
    (dict(Tspan=np.inf), "Tspan"),
    (dict(log10_A_common=np.nan), "log10_A_common"),
    (dict(log10_A_common=-14.0, gamma_common=np.inf), "gamma_common"),
    (dict(log10_A_common=-14.0, components_common=0), "components_common"),
])
def test_argument_checks(kw, match):
    b = _batch(_small())
    with pytest.raises(ValueError, match=match):
        b.set_red_noise_likelihood(**kw)


def test_missing_white_noise_raises_in_plan():
    b = _batch(_small(), white=False)
    b.set_red_noise_likelihood()
    with pytest.raises(ValueError, match="red-noise likelihood needs white noise"):
        b.plan()


def test_non_psd_z_raises_naming_pulsar_and_gamma(monkeypatch):
    """A Z_a that is negative definite (C_a negated for pulsar 1 only) is refused, naming that pulsar and the first gamma."""
    b = _batch(_small())
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=4)
    pinv = b._pinv_apply
    monkeypatch.setattr(b, "_pinv_apply", lambda i, *a, **k: -pinv(i, *a, **k) if i == 1 else pinv(i, *a, **k))
    with pytest.raises(ValueError, match=r"Z_a of pulsar 1 \(.*\) is not positive semi-definite at gamma = 2.0"):
        b.plan()


def test_pulsar_without_span_needs_tspan():
    b = _batch(_small())
    b.t_tdb[2] = np.full_like(b.t_tdb[2], b.t_tdb[2][0])
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=2)
    with pytest.raises(ValueError, match="pulsar 2 .* spans no time"):
        b.plan()
