"""Per-realization common-process populations on the device (``set_common_population``, ``ptar_common_population``):
the draws against the numpy restatement of tests/cpop_oracle.py, the injection against F_a c_a on the host (noise and
alignment slots untouched), chunk / real0 / shard invariance, composition with the CW population and the timing fit,
refusals, and the calibration of the CURN, HD and free-spectrum posteriors (simulation-based calibration: the posterior
rank of the injected value is Uniform(0, 1)) with a negative control that shows the test has power."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

from tests import cpop_oracle as PO
from tests import generator_reference as GR
from tests.reduction_reference import EDGE_NTOAS, U

pytestmark = pytest.mark.gpu

SEED = 20261018
KS_PASS = 1e-3          # calibration: p-value of KS against Uniform(0, 1) above this
KS_FAIL = 1e-6          # negative control: p-value below this


def _np(t):
    return t.detach().cpu().numpy()


def _batch(P, ntoas=None, **kw):
    """Dense edge pulsars (odd TOA counts, epochs straddling tiles) with white noise."""
    from pta_replicator_b200.engine import PulsarBatch
    pool = GR.GEN_NTOAS + EDGE_NTOAS
    ntoas = ntoas or {1: (1025,), 3: (1, (17, 2), 2100)}.get(P) or tuple(pool[j % len(pool)] for j in range(P))
    b = PulsarBatch(GR.dense_pulsars(ntoas, seed=P, name="Q"), **kw)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.0, log10_equad=-6.5)
    return b


def _slots(b):
    sel = np.concatenate([np.arange(o, o + n) for o, n in zip(b.toa_off, b.ntoa)])
    pad = np.ones(b.ld, dtype=bool)
    pad[sel] = False
    return sel, pad


# ------------------------------------------------------------------ draws
@pytest.mark.parametrize("case", [dict(orf="hd", components=14), dict(orf=None, components=3, gamma=(1.0, 6.0)),
                                  dict(orf="monopole", components=32, log10_A=-14.5),
                                  dict(spectrum="free", orf="dipole", components=9),
                                  dict(spectrum="free", orf=None, components=1, log10_rho=-7.0)])
def test_params_equal_numpy_restatement(case):
    """Hyperparameters bit for bit (the affine map); coefficients within 32 u of sqrt(phi) sum_b |B_ab| |z_b| (the
    normals' log / sincos, 10^x and pow differ from numpy's by a few ulp; the mixing's order is the same)."""
    b = _batch(5)
    b.set_common_population(**case)
    R, r0 = 300, 1001
    got = {k: _np(v) for k, v in b.common_population_params(R, seed=SEED, real0=r0, coefficients=True).items()}
    rr = np.arange(r0, r0 + R)
    hyp = PO.hyper(b._cpop, rr, SEED)
    for k, v in hyp.items():
        assert np.array_equal(got[k], v), k
    c, env, _ = PO.coefficients(b._cpop, rr, SEED, b.n_psr)
    d = np.abs(got["c"] - c)
    ratio = np.max(d / (32 * U * env))
    print(f"\n[cpop] {case}: max |dc| / (32 u envelope) = {ratio:.3f}")
    assert ratio <= 1.0
    assert got["c"].shape == (R, b.n_psr, 2 * b._cpop["K"])


# ------------------------------------------------------------------ injection
@pytest.mark.parametrize("P", (1, 3))
def test_injection_equals_host_basis(P):
    """rows with - rows without a population = F_a c_a on the host (from the returned c and _sincos_basis) within
    1e-12 of the injection's rms, every bin-count template (K = 1, 9, 17, 32), with the pre-filled alignment slots
    (NaN) untouched."""
    import torch
    b = _batch(P)
    R = 37                                                       # not a multiple of the add kernel's realization block
    sel, pad = _slots(b)

    def rows():
        out = torch.full((R, b.ld), float("nan"), dtype=torch.float64, device=b.device)
        return _np(b.generate(R, seed=SEED, out=out))

    without = rows()
    for K, orf, spectrum in ((1, None, "powerlaw"), (9, "hd", "free"), (17, "monopole", "powerlaw"), (32, "hd", "powerlaw")):
        if orf is not None and P == 1 and orf != "monopole":
            orf = None
        b.set_common_population(components=K, orf=orf, spectrum=spectrum, log10_A=(-13.5, -12.5), log10_rho=(-7.0, -6.0))
        with_ = rows()
        assert np.array_equal(with_[:, pad], without[:, pad], equal_nan=True)          # alignment slots untouched
        assert np.isfinite(with_[:, sel]).all()
        c = _np(b.common_population_params(R, seed=SEED, coefficients=True)["c"])
        inj = PO.injection(b, c, K, b._cpop["Tspan"])
        rms = np.sqrt(np.mean(inj[:, sel] ** 2))
        err = np.max(np.abs((with_ - without)[:, sel] - inj[:, sel]))
        print(f"\n[cpop] P={P} K={K} orf={orf} {spectrum}: max |(with - without) - F c| = {err / rms:.2e} of the rms")
        assert err <= 1e-12 * rms
    b.set_common_population(None)
    assert np.array_equal(rows(), without, equal_nan=True)


# ------------------------------------------------------------------ invariance
def test_chunk_real0_and_shard_invariance():
    import torch
    from pta_replicator_b200 import distributed
    b = _batch(3, ntoas=(65, 193, 1025))
    b.set_common_population(components=20)
    N = 40
    full = b.generate(N, seed=SEED, chunk=8)
    part = b.generate(16, seed=SEED, real0=8, chunk=12)
    assert torch.equal(full[8:24], part)
    for world in (2, 3):
        for rank in range(world):
            s, n = distributed.shard_bounds(N, world, rank)
            if n:
                assert torch.equal(b.generate(n, seed=SEED, real0=s), full[s:s + n]), (world, rank)
    pf = b.common_population_params(N, seed=SEED, coefficients=True)
    pp = b.common_population_params(16, seed=SEED, real0=8, coefficients=True)
    for k in pf:
        assert torch.equal(pf[k][8:24], pp[k]), k


# ------------------------------------------------------------------ composition
def test_with_cw_population():
    b = _batch(3)
    R = 12
    sel, _ = _slots(b)
    none = _np(b.generate(R, seed=SEED))
    b.set_common_population(components=6, log10_A=-13.0)
    cp = _np(b.generate(R, seed=SEED))
    b.set_cw_population(n_sources=2, log10_h0=-13.5)
    both = _np(b.generate(R, seed=SEED))
    b.set_common_population(None)
    cw = _np(b.generate(R, seed=SEED))
    d = (both - none) - ((cp - none) + (cw - none))
    scale = np.max(np.abs(both))
    print(f"\n[cpop] with the CW population: max |additivity defect| = {np.max(np.abs(d[:, sel])):.2e} of {scale:.2e}")
    assert np.max(np.abs(d[:, sel])) <= 1e-13 * scale


def test_timing_fit_projects_the_injection():
    import torch
    from pta_replicator_b200 import _cabi
    b = _batch(3, ntoas=(65, 193, 1025))
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    R = 8
    post0 = b.generate(R, seed=SEED)
    pre0 = b._generate(R, SEED, 0, None, None, None, 0, None, postfit=False).clone()
    b.set_common_population(components=10, log10_A=-13.0)
    post1 = b.generate(R, seed=SEED)
    pre1 = b._generate(R, SEED, 0, None, None, None, 0, None, postfit=False).clone()
    inj = (pre1 - pre0).contiguous()
    scale = float(inj.abs().max())
    assert scale > 0
    tm = b.compile()["tm"]
    scratch = torch.empty(tm["n_tiles"] * R * tm["kmax"], dtype=torch.float64, device=b.device)
    _cabi.check(_cabi.lib().ptar_timing_project(inj.data_ptr(), b.ld, R, C.addressof(tm["model"]), scratch.data_ptr(),
                                                scratch.numel(), _cabi.current_stream()), "ptar_timing_project")
    err = float(((post1 - post0) - inj).abs().max())
    print(f"\n[cpop] timing fit: max |(post-fit with - without) - fit(injection)| = {err:.3e} of {scale:.3e}")
    assert err <= 1e-12 * scale


def test_removal_and_refusals():
    import torch
    b = _batch(3)
    ref = b.generate(8, seed=SEED)
    b.set_common_population(components=4)
    assert not torch.equal(b.generate(8, seed=SEED), ref)
    with pytest.raises(ValueError, match="common-process"):
        b.generate(8, inject=dict(z1=torch.zeros(8, b.ld), z2=torch.zeros(8, b.ld)))
    with pytest.raises(ValueError, match="generate"):
        b.generate_to_host(8, seed=SEED)
    b.set_common_population(None)
    assert torch.equal(b.generate(8, seed=SEED), ref)
    with pytest.raises(ValueError):
        b.common_population_params(8)


# ------------------------------------------------------------------ calibration
X_CAL = np.linspace(-15.5, -13.0, 121)        # log10 A grid and prior
G_CAL = np.linspace(2.0, 6.0, 81)             # gamma grid and prior
RHO_CAL = np.linspace(-10.0, -4.0, 241)       # log10 rho grid and prior (free spectrum)
R_CAL = 2048
SHIFT = 0.25                                  # negative control: the injected value shifted by this much


def _ks(ranks):
    return stats.kstest(np.asarray(ranks, dtype=float), "uniform").pvalue


def _ng15_cal():
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("full", npsr=10)
    return synthetic.ng15_recipe(PulsarBatch(psrs), noise, gwb=False)


def test_calibration_curn_hd_free_spectrum():
    """Simulation-based calibration on 10 ng15-full pulsars (white noise, ECORR, red noise, no GWB), priors equal to
    the grids: the posterior CDF at the injected value, over 2048 realizations, passes KS against Uniform(0, 1) for
    (a) log10 A and gamma of CURN with an uncorrelated population, (b) of HD with an HD population, (c) log10 rho of
    the free spectrum at one bin, where the factorised likelihood is exact; (d) the same ranks at the injected value
    shifted by 0.25 fail it.  The K = 14 free-spectrum coverage is printed, not asserted (its bins couple)."""
    from pta_replicator_b200.engine import grid_cdf
    b = _ng15_cal()
    b.set_curn_likelihood(log10_A=X_CAL, gamma=G_CAL, components=14)
    b.set_hd_likelihood()
    report = []

    def check(name, post, grid, truth):
        p = _ks(_np(grid_cdf(post, grid, truth)))
        p_neg = _ks(_np(grid_cdf(post, grid, truth + SHIFT)))
        report.append(f"{name}: KS p = {p:.3g}, shifted by {SHIFT}: {p_neg:.3g}")
        assert p > KS_PASS, report[-1]
        assert p_neg < KS_FAIL, report[-1]

    for orf, pre in ((None, ""), ("hd", "hd_")):
        b.set_common_population(log10_A=(X_CAL[0], X_CAL[-1]), gamma=(G_CAL[0], G_CAL[-1]), components=14, orf=orf)
        res = b.curn_likelihood(R_CAL, seed=SEED)
        tru = b.common_population_params(R_CAL, seed=SEED)
        check(f"{pre or 'curn_'}log10_A", res[pre + "post_log10_A"], X_CAL, tru["log10_A"])
        check(f"{pre or 'curn_'}gamma", res[pre + "post_gamma"], G_CAL, tru["gamma"])
        ulp = grid_cdf(res[pre + "post_log10_A"], X_CAL, res[pre + "log10_A_ul"])      # the upper limit's quantile
        assert float((ulp - 0.95).abs().max()) <= 1e-9
        hit = _np(res[pre + "log10_A_ul"] >= tru["log10_A"]).mean()
        report.append(f"{pre or 'curn_'}log10_A_ul covers the injection in {hit:.3f} of {R_CAL}")
    b.set_free_spectrum(log10_rho=RHO_CAL, components=1)
    b.set_common_population(spectrum="free", components=1, log10_rho=(RHO_CAL[0], RHO_CAL[-1]), orf=None)
    res = b.free_spectrum(R_CAL, seed=SEED)
    tru = b.common_population_params(R_CAL, seed=SEED)["log10_rho"]
    check("fs K=1 log10_rho", res["post_log10_rho"][:, 0], RHO_CAL, tru[:, 0])
    # K = 14: the factorised free spectrum leaves out the coupling between bins, so its coverage is reported only
    b.set_free_spectrum(log10_rho=RHO_CAL, components=14)
    b.set_common_population(spectrum="free", components=14, log10_rho=(RHO_CAL[0], RHO_CAL[-1]), orf=None)
    res = b.free_spectrum(1024, seed=SEED + 1)
    tru = b.common_population_params(1024, seed=SEED + 1)["log10_rho"]
    ps = [_ks(_np(grid_cdf(res["post_log10_rho"][:, k], RHO_CAL, tru[:, k]))) for k in range(14)]
    report.append("fs K=14 per-bin KS p (not asserted): " + ", ".join(f"{p:.2g}" for p in ps))
    print("\n[cpop calibration] " + "\n[cpop calibration] ".join(report))
