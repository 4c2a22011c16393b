"""Common-process populations on the host: the Philox stream of kind 8 (tests/cpop_oracle.py) against Philox4x32-10
itself and the other streams, the laws of the hyperparameters, the fp64 normals and the coefficients (KS tests, moments,
covariance against A^2 Gamma (x) phi~), the spectrum against ``_powerlaw_prior``, the argument checks of
``set_common_population`` on a plan-only batch, and ``grid_cdf`` against closed forms and as the inverse of the
device's upper-limit convention on tests/summary_reference.py's summaries."""
import numpy as np
import pytest
import torch
from scipy import stats

from oracle.philox import philox4x32_10
from tests import cpop_oracle as PO
from tests import cwpop_oracle as CO
from tests import generator_reference as GR
from tests import summary_reference as SR

SEED = 0x51ED5EED0042


def _batch(ntoas=(7, 33, 64, 20, 41), **kw):
    from pta_replicator_b200.engine import PulsarBatch
    return PulsarBatch(GR.dense_pulsars(ntoas, seed=5, name="C"), plan_only=True, **kw)


def _blocks(w):
    """The 128-bit outputs of Philox calls (4 words each) as one comparable key per call."""
    a = np.ascontiguousarray(np.stack([np.broadcast_to(x, np.broadcast(*w).shape).ravel() for x in w], axis=1)
                             .astype(np.uint32))
    return a.view(np.dtype((np.void, 16))).ravel()


# ------------------------------------------------------------------ the stream
def test_words_are_philox_at_the_documented_counters():
    elem = np.array([0, 1, 13, 31, PO.HYPER, PO.HYPER + 15])
    for psr in (0, 1, 66, 2047):
        for r in (0, 1, 7, 2**32 + 5, 2**40 + 3):
            w = PO.words(elem, psr, r, SEED)
            ref = philox4x32_10(elem, 8 | (psr << 8), r & 0xFFFFFFFF, r >> 32, SEED)
            for a, b in zip(w, ref):
                assert np.array_equal(a, b)


def test_hyper_pairs_and_word_halves():
    """Hyperparameter j takes pair j // 2 and words (x, y) for even j, (z, w) for odd j."""
    r = np.arange(50)
    for j in range(6):
        w = PO.words(PO.HYPER + j // 2, 0, r, SEED)
        want = CO.uniform53(w[0], w[1]) if j % 2 == 0 else CO.uniform53(w[2], w[3])
        assert np.array_equal(PO._hyper_uniform(j, r, SEED), want)


def test_no_collision_with_other_streams():
    r = np.arange(64)[:, None]
    mine = np.concatenate([_blocks(PO.words(np.arange(32), p, r, SEED)) for p in (0, 5)]
                          + [_blocks(PO.words(PO.HYPER + np.arange(16), 0, r, SEED))])
    assert np.unique(mine).size == mine.size
    for kind in range(1, 8):
        for rf in (r, r >> 2):          # the noise streams key (c.z, c.w) on r >> 2, the CW population on r
            for p in (0, 5):
                w = _blocks(philox4x32_10(np.r_[0:512, PO.HYPER:PO.HYPER + 16], kind | (p << 8), rf, 0, SEED))
                assert np.intersect1d(mine, w).size == 0, kind


# ------------------------------------------------------------------ laws
def _pop(b, **kw):
    b.set_common_population(**kw)
    return b._cpop


def test_hyperparameter_laws_ks():
    b = _batch()
    pop = _pop(b, log10_A=(-16.0, -13.0), gamma=(1.0, 6.0), orf=None)
    h = PO.hyper(pop, np.arange(100_000), SEED)
    for name, x in (("log10_A", (h["log10_A"] + 16) / 3), ("gamma", (h["gamma"] - 1) / 5)):
        p = stats.kstest(x, "uniform").pvalue
        assert p > 1e-3, (name, p)
        assert x.min() >= 0 and x.max() < 1
    assert abs(stats.pearsonr(h["log10_A"], h["gamma"])[0]) < 0.02
    pop = _pop(b, spectrum="free", log10_rho=(-9.0, -5.0), components=5)
    h = PO.hyper(pop, np.arange(40_000), SEED)["log10_rho"]
    assert h.shape == (40_000, 5)
    for k in range(5):
        assert stats.kstest((h[:, k] + 9) / 4, "uniform").pvalue > 1e-3, k
    c = np.corrcoef(h.T)
    assert np.max(np.abs(c - np.eye(5))) < 0.03                       # independent bins


def test_fixed_hyperparameters_exact():
    b = _batch()
    h = PO.hyper(_pop(b, log10_A=-14.123456789, gamma=13 / 3), np.arange(64), SEED)
    assert np.all(h["log10_A"] == -14.123456789) and np.all(h["gamma"] == 13 / 3)
    h = PO.hyper(_pop(b, spectrum="free", log10_rho=-7.5, components=3), np.arange(64), SEED)
    assert np.all(h["log10_rho"] == -7.5)


def test_normals_ks_and_moments():
    z = PO.normals(np.arange(4000), 5, 4, SEED).ravel()               # 160,000 normals
    assert stats.kstest(z, "norm").pvalue > 1e-3
    n = z.size
    # sample moments to order 4 against N(0, 1): E z = 0, E z^2 = 1, E z^3 = 0, E z^4 = 3 (standard errors from the
    # moments of order 2, 4, 6 and 8: 1, 2, 15, 96)
    for order, mean, var in ((1, 0.0, 1.0), (2, 1.0, 2.0), (3, 0.0, 15.0), (4, 3.0, 96.0)):
        zz = (np.mean(z**order) - mean) / np.sqrt(var / n)
        assert abs(zz) < 5, (order, zz)
    pairs = PO.normals(np.arange(4000), 2, 2, SEED)
    assert abs(np.corrcoef(pairs[..., 0].ravel(), pairs[..., 1].ravel())[0, 1]) < 0.02   # sin / cos of one pair


@pytest.mark.parametrize("orf", ("hd", "monopole"))
def test_coefficient_covariance(orf):
    """At fixed (A, gamma): Cov(c[a, j], c[b, j]) = A^2 Gamma_ab phi~_j, each entry within 5 sigma of its estimate's
    spread (Gamma_aa Gamma_bb + Gamma_ab^2) phi~_j^2 A^4 / R."""
    from pta_replicator_b200.engine import _powerlaw_prior
    b = _batch()
    la, g, K = -14.0, 3.0, 3
    pop = _pop(b, log10_A=la, gamma=g, components=K, orf=orf)
    R = 40_000
    c, _, _ = PO.coefficients(pop, np.arange(R), SEED, b.n_psr)
    G = pop["orf"]["orf"]
    pt = _powerlaw_prior(np.arange(1, K + 1) / pop["Tspan"], g, pop["Tspan"])
    worst = 0.0
    for j in range(2 * K):
        S = c[:, :, j].T @ c[:, :, j] / R
        want = 10.0 ** (2 * la) * G * pt[j]
        sd = 10.0 ** (2 * la) * pt[j] * np.sqrt((np.outer(np.diag(G), np.diag(G)) + G**2) / R)
        zz = np.abs(S - want) / sd
        worst = max(worst, zz.max())
    print(f"\n[cpop] {orf}: worst |covariance - A^2 Gamma phi~| = {worst:.2f} sigma")
    assert worst < 5
    if orf == "monopole":   # rank 1: every pulsar carries the same process, up to the square roots (~ sqrt(u)) of the
        # eigen factor's rounding-level eigenvalues, which change Gamma = B B^T itself only at rounding
        assert np.max(np.abs(c - c[:, :1, :])) <= 1e-6 * np.max(np.abs(c))
        assert np.allclose(pop["orf"]["B"] @ pop["orf"]["B"].T, G, rtol=0, atol=1e-14)


def test_spectrum_matches_powerlaw_prior_and_free_convention():
    from pta_replicator_b200.engine import _powerlaw_prior
    b = _batch()
    pop = _pop(b, components=7)
    h = PO.hyper(pop, np.arange(200), SEED)
    a = PO.amplitude(pop, h)
    f = np.arange(1, 8) / pop["Tspan"]
    for r in range(200):
        want = 10.0 ** (2 * h["log10_A"][r]) * _powerlaw_prior(f, h["gamma"][r], pop["Tspan"])[0::2]
        np.testing.assert_allclose(a[r] ** 2, want, rtol=1e-14)
    pop = _pop(b, spectrum="free", components=4)
    h = PO.hyper(pop, np.arange(200), SEED)
    np.testing.assert_allclose(PO.amplitude(pop, h) ** 2, 10.0 ** (2 * h["log10_rho"]), rtol=1e-15)


# ------------------------------------------------------------------ registration
def test_registration_defaults_and_removal():
    from pta_replicator_b200 import _cabi
    b = _batch()
    assert b._cpop is None
    b._compiled = "x"
    b.set_common_population()
    assert b._compiled is None
    cp = b._cpop
    assert cp["K"] == 14 and cp["spectrum"] == "powerlaw" and cp["orf"]["name"] == "hd"
    assert cp["kind"] == [_cabi.CWPOP_UNIFORM] * 2 and cp["lo"] == [-18.0, 0.0] and cp["width"] == [6.0, 7.0]
    assert cp["Tspan"] == b._array_tspan(None)
    b.set_curn_likelihood()
    b.set_free_spectrum()
    assert (cp["lo"][0], cp["lo"][0] + cp["width"][0]) == (b._curn["log10_A"][0], b._curn["log10_A"][-1])
    assert (cp["lo"][1], cp["lo"][1] + cp["width"][1]) == (b._curn["gamma"][0], b._curn["gamma"][-1])
    b.set_common_population(spectrum="free", orf=None, log10_A="ignored", gamma=None)   # the power law's are ignored
    cp = b._cpop
    assert cp["orf"] is None and cp["kind"][0] == _cabi.CWPOP_UNIFORM
    assert (cp["lo"][0], cp["lo"][0] + cp["width"][0]) == (b._fs["log10_A"][0], b._fs["log10_A"][-1])   # its log10 rho grid
    b.set_common_population(orf=np.eye(b.n_psr), Tspan=4e8, components=32)
    assert b._cpop["orf"]["name"] == "matrix" and b._cpop["Tspan"] == 4e8 and b._cpop["K"] == 32
    b.set_common_population(orf="monopole")
    assert np.allclose(b._cpop["orf"]["B"] @ b._cpop["orf"]["B"].T, np.ones((b.n_psr, b.n_psr)))
    b._compiled = "x"
    b.set_common_population(None)
    assert b._cpop is None and b._compiled is None


@pytest.mark.parametrize("kw", [
    dict(log10_A=(-12.0, -18.0)), dict(log10_A=(-14.0, -14.0)), dict(gamma=(1.0,)), dict(gamma=(1, 2, 3)),
    dict(log10_A=float("nan")), dict(gamma=(0.0, float("inf"))), dict(gamma=None), dict(log10_A="x"),
    dict(log10_A=400.0), dict(log10_A=(-14.0, 170.0)), dict(gamma=(0.0, 250.0)),
    dict(spectrum="free", log10_rho=(-4.0, -10.0)), dict(spectrum="free", log10_rho=float("-inf")),
    dict(spectrum="free", log10_rho=None), dict(spectrum="free", log10_rho=(1.0, 2.0, 3.0)),
    dict(components=0), dict(components=33), dict(components=1.5), dict(components=True),
    dict(spectrum="turnover"), dict(spectrum=None), dict(orf="quadrupole"), dict(orf=-np.eye(5)),
    dict(orf=np.ones((4, 4))), dict(orf=np.diag([1.0, 1.0, 1.0, 1.0, -0.5])),
    dict(orf=np.array([[1.0, 0.9, 0, 0, 0], [0.1, 1, 0, 0, 0], [0, 0, 1, 0, 0], [0, 0, 0, 1, 0], [0, 0, 0, 0, 1]])),
    dict(Tspan=0.0), dict(Tspan=-1.0), dict(Tspan=float("nan")),
])
def test_bad_arguments_raise(kw):
    b = _batch()
    with pytest.raises(ValueError):
        b.set_common_population(**kw)
    assert b._cpop is None


def test_plan_only_device_calls_raise():
    from pta_replicator_b200 import _cabi
    b = _batch()
    b.set_common_population(components=4)
    b.plan()
    with pytest.raises(_cabi.PtarError):
        b.common_population_params(8)
    with pytest.raises(_cabi.PtarError):
        b.common_population_params(8, coefficients=True)
    with pytest.raises(_cabi.PtarError):
        b.generate(8)


# ------------------------------------------------------------------ grid_cdf
def test_grid_cdf_closed_forms():
    from pta_replicator_b200.engine import grid_cdf
    x = np.linspace(0.0, 1.0, 11)
    uni = torch.ones(3, 11, dtype=torch.float64)
    q = torch.tensor([0.0, 0.37, 1.0], dtype=torch.float64)
    assert torch.allclose(grid_cdf(uni, x, q), q, rtol=0, atol=1e-15)
    assert torch.equal(grid_cdf(uni, x, torch.tensor([-0.5, 1.5, float("nan")])).isnan(), torch.tensor([False, False, True]))
    assert grid_cdf(uni, x, -0.5)[0] == 0.0 and grid_cdf(uni, x, 1.5)[0] == 1.0
    # triangular density 2x: trapezoid is exact for a linear density, so the CDF is x^2 at the nodes and linear between
    tri = torch.from_numpy(2 * x)[None].repeat(2, 1)
    assert torch.allclose(grid_cdf(tri, x, torch.from_numpy(x)[:, None].expand(11, 2)), torch.from_numpy(x**2)[:, None],
                          rtol=0, atol=1e-15)
    v = 0.43                                                            # off the nodes: between 0.4 and 0.5
    want = 0.16 + (v - 0.4) / 0.1 * (0.25 - 0.16)
    assert abs(float(grid_cdf(tri, x, v)[0]) - want) < 1e-15
    # an unnormalised density and a non-uniform grid: normalised by the last node
    g = np.array([-3.0, -2.5, -1.0, 0.5, 2.0])
    p = torch.tensor([[0.0, 2.0, 4.0, 2.0, 0.0]], dtype=torch.float64)
    w = 0.5 * np.diff(g) * (p[0, 1:] + p[0, :-1]).numpy()
    cdf = np.r_[0, np.cumsum(w)] / w.sum()
    assert torch.allclose(grid_cdf(p, g, torch.from_numpy(g)[:, None]).ravel(), torch.from_numpy(cdf), rtol=0, atol=1e-15)
    with pytest.raises(ValueError):
        grid_cdf(uni, x[:5], 0.5)
    with pytest.raises(ValueError):
        grid_cdf(uni[:, :1], x[:1], 0.5)


def test_grid_cdf_inverts_the_upper_limit():
    """On the constructed maps of tests/summary_reference.py, at every ul, grid_cdf of the posterior at the reference's
    upper limit is ul, to the reference's own upper-limit bound times the density there (where the CDF rises)."""
    from pta_replicator_b200.engine import grid_cdf
    worst, n = 0.0, 0
    for NA, NG in ((97, 57), (64, 5), (3, 2)):
        for spacing in ("uniform", "geometric"):
            x, g = SR.grid(NA, NG, spacing)
            st = SR.statics(x, g, "log-uniform")
            _, maps = SR.curn_maps(x, g)
            for ul in SR.ULS:
                out = SR.curn_summaries(maps, st["log10_A"], st["gamma"], st["wg"], st["wx"], st["prior"], ul)
                post, lim = out["post_log10_A"]["hi"], out["log10_A_ul"]
                ok = np.isfinite(lim["hi"])
                got = grid_cdf(torch.from_numpy(post[ok]), x, torch.from_numpy(lim["hi"][ok])).numpy()
                # the density at the limit bounds how far the CDF moves within the limit's tolerance
                k = np.clip(np.searchsorted(x, lim["hi"][ok]), 1, NA - 1)
                dens = np.maximum(post[ok, k - 1], post[ok, k]) / np.sum(0.5 * np.diff(x) * (post[ok, 1:] + post[ok, :-1]),
                                                                         axis=1)
                tol = dens * lim["bound"][ok] + 1e-12
                err = np.abs(got - ul)
                assert np.all(err <= tol), (NA, NG, spacing, ul, np.max(err / tol))
                worst = max(worst, float(np.max(err)))
                n += int(ok.sum())
    print(f"\n[grid_cdf] {n} upper limits: max |grid_cdf(post, grid, ul_value) - ul| = {worst:.2e}")
