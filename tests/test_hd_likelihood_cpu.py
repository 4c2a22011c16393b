"""CPU tests of the HD likelihood's host statics (``PulsarBatch.set_hd_likelihood``, ``plan()["hd"]``) against the dense
stacked-covariance oracle (tests/hd_oracle.py), its reduction to CURN at Gamma = I, the isolation of the other
statistics' statics and the argument checks.  ``plan_only`` batches: the 3 ``partim_small`` pulsars and the 4-pulsar
synthetic case of the optimal-statistic tests, with and without a timing model, for the named templates and a random
positive semi-definite matrix."""
import numpy as np
import pytest

from tests import curn_oracle as CO
from tests import hd_oracle as HO
from tests import os_oracle as OO
from tests.test_curn_likelihood_cpu import G_GRID, TOL, X_GRID, _rows
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic


def _psd(P, seed=0, rank=None):
    """A random symmetric positive semi-definite [P, P] matrix (rank ``rank``, default full), diagonal not 1."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((P, P if rank is None else rank))
    return A @ A.T / P


CASES = [(src, tm, orf) for src in ("small", "synthetic") for tm in (False, True)
         for orf in ("hd", "monopole", "dipole", "psd")]


@pytest.mark.parametrize("src,tm,orf", CASES)
def test_statics_match_dense_oracle(src, tm, orf):
    psrs = _small() if src == "small" else _synthetic()
    b = _batch(psrs, tm=tm)
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    o = _psd(b.n_psr, seed=len(psrs)) if orf == "psd" else orf
    b.set_hd_likelihood(orf=o)
    pl = b.plan()
    pc, ph = pl["curn"], pl["hd"]
    rows = _rows(b, 5, seed=len(psrs))
    got = HO.lnl_of_statics(b, pc, ph, rows)
    ref, ld = HO.lnl_map(b, rows, X_GRID, G_GRID, orf=o, K=6, models=_models(b) if tm else None)
    d = float(np.max(np.abs(got - ref)))
    dl = float(np.max(np.abs(ph["ldet"] - ld) / np.maximum(1.0, np.abs(ld))))
    print(f"\n[hd] {src} tm={tm} orf={orf}: max |d lnL| = {d:.1e} (|lnL| <= {np.max(np.abs(ref)):.1e}), "
          f"ldet rel {dl:.1e}")
    assert d <= TOL and dl <= 1e-9
    N = b.n_psr * 12
    assert ph["n"] == N and ph["np"] == -(-N // 32) * 32 and ph["V"].shape == (3, ph["np"], b.n_psr * 16)
    V = ph["V"].reshape(3, ph["np"], b.n_psr, 16)
    assert np.all(V[:, N:] == 0) and np.all(V[..., 12:] == 0) and np.all(ph["lam"][:, N:] == 0)
    assert np.all(ph["eig"] >= 0) and ph["eig"].shape == (3, N)
    if orf == "monopole":   # rank-1 Gamma: at most nc nonzero eigenvalues per gamma
        assert np.all(np.sum(ph["eig"] > 1e-12 * ph["eig"].max(axis=1, keepdims=True), axis=1) <= 12)


@pytest.mark.parametrize("src,tm", [("small", True), ("synthetic", False)])
def test_identity_orf_reduces_to_curn(src, tm):
    psrs = _small() if src == "small" else _synthetic()
    b = _batch(psrs, tm=tm)
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    b.set_hd_likelihood(orf=np.eye(b.n_psr))
    pl = b.plan()
    rows = _rows(b, 5, seed=7)
    hd = HO.lnl_of_statics(b, pl["curn"], pl["hd"], rows)
    cu = CO.lnl_of_statics(b, pl["curn"], rows)
    rel = float(np.max(np.abs(hd - cu)) / np.max(np.abs(cu)))
    print(f"\n[hd] Gamma = I vs CURN, {src} tm={tm}: max |d lnL| / max |lnL| = {rel:.1e}")
    assert rel <= 1e-10
    np.testing.assert_allclose(pl["hd"]["ldet"], pl["curn"]["ldet"], rtol=1e-10)
    np.testing.assert_allclose(np.sort(pl["hd"]["eig"], axis=1),
                               np.sort(pl["curn"]["eig"].transpose(1, 0, 2).reshape(3, -1), axis=1),
                               rtol=1e-9, atol=1e-12 * pl["curn"]["eig"].max())


def test_registration_leaves_other_statistics_unchanged():
    b = _batch(_small(), tm=True)
    b.set_optimal_statistic()
    b.set_fp_statistic(n_freqs=5)
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID)
    pl0 = b.plan()
    assert pl0["hd"] is None and b.hd_setup_s is None
    b.set_hd_likelihood()
    pl1 = b.plan()
    for sec in ("curn", "os", "fp"):
        for k, v in pl0[sec].items():
            if k != "setup_s":
                assert np.array_equal(np.asarray(v), np.asarray(pl1[sec][k])), (sec, k)
    assert pl1["hd"]["setup_s"] > 0 and b.hd_setup_s == pl1["hd"]["setup_s"]
    assert pl1["hd"]["name"] == "hd"
    np.testing.assert_allclose(pl1["hd"]["orf"], OO.hd_closed_form(b)[0], rtol=1e-9, atol=1e-12)
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID)     # a new CURN registration drops the HD one
    assert b.plan()["hd"] is None


def test_named_templates_spectra():
    """The ORF eigenvalues the statics use: HD positive definite, monopole rank 1, dipole rank <= 3 (clipped)."""
    b = _batch(_synthetic())
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    for orf, rank in (("hd", 4), ("monopole", 1), ("dipole", 3)):
        b.set_hd_likelihood(orf=orf)
        mu = b._hd["mu"]
        assert np.all(mu >= 0) and np.sum(mu > 1e-10 * mu[-1]) <= rank, (orf, mu)
    b.set_hd_likelihood(orf=_psd(4, rank=2))                  # rank-deficient matrices are accepted
    assert np.sum(b._hd["mu"] > 1e-10 * b._hd["mu"][-1]) == 2


def _bad_matrices():
    G = _psd(3, seed=1)
    asym = G.copy()
    asym[0, 1] += 1e-3
    nan = G.copy()
    nan[1, 1] = np.nan
    inf = G.copy()
    inf[0, 2] = inf[2, 0] = np.inf
    neg = np.diag([1.0, 1.0, -1e-3])                          # mu_min / mu_max = -1e-3
    return [(asym, "symmetric"), (nan, "finite"), (inf, "finite"), (np.eye(4), r"\[3, 3\]"), (np.eye(3)[:, :2], r"\[3, 3\]"),
            (neg, "positive semi-definite"), (-np.eye(3), "positive semi-definite"), ("quadrupole", "unknown ORF")]


@pytest.mark.parametrize("orf,match", _bad_matrices())
def test_argument_checks(orf, match):
    b = _batch(_small())
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID)
    with pytest.raises(ValueError, match=match):
        b.set_hd_likelihood(orf=orf)
    assert b._hd is None


def test_needs_curn_registration_and_two_pulsars():
    b = _batch(_small())
    with pytest.raises(ValueError, match="no CURN likelihood registered"):
        b.set_hd_likelihood()
    one = _batch(_small()[:1])
    one.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID)
    with pytest.raises(ValueError, match="at least 2 pulsars"):
        one.set_hd_likelihood()


def test_size_limit():
    """N = n_psr 2K <= 4096: 128 pulsars at K = 16 is the largest batch, 129 pulsars is refused."""
    from pta_replicator_b200.engine import PulsarBatch
    from tests import reduction_reference as RR
    psrs = RR.edge_pulsars((5,) * 129, seed=3)
    big = PulsarBatch(psrs, plan_only=True)
    big.set_curn_likelihood(components=16)
    with pytest.raises(ValueError, match="N = 4128"):
        big.set_hd_likelihood()
    big.set_curn_likelihood(components=15)                  # N = 3870
    big.set_hd_likelihood()
    ok = PulsarBatch(psrs[:128], plan_only=True)
    ok.set_curn_likelihood(components=16)                   # N = 4096
    ok.set_hd_likelihood()
