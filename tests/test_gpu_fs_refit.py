"""GPU tests of the free spectrum's spectral refit (``PulsarBatch.set_spectral_refit`` -> ``ptar_os_project`` +
``ptar_fs_y2`` + ``ptar_fs_refit`` + ``ptar_curn_reduce``): edge shapes against an extended-precision evaluation with a
rounding bound and alignment slots holding NaN and +-inf, the tie to the tested free-spectrum kernel at grid nodes, the
tie to the CURN and HD kernels at one bin, the device against numpy on the plan's statics and against the dense refit
oracle, the summaries against numpy on the device's own maps under both priors, bit-identity across chunking, real0
splits, maps, paths and map sub-blocks (and of the free spectrum's own outputs with and without a refit), the exact mean
of Q under the noise model, and the recovery of loud power-law and turnover injections of ``set_gwb``."""
import numpy as np
import pytest

from pta_replicator_b200 import spectra
from tests import curn_oracle as CO
from tests import fs_refit_oracle as RO
from tests import reduction_reference as RR
from tests.test_gpu_curn_likelihood import _ng15, _small_tm
from tests.test_gpu_hd_likelihood import _ng15_epoch
from tests.test_gpu_reduction_edges import _equal, _np, _poison, _rows, _t

pytestmark = pytest.mark.gpu

SEED = 20261018
KEYS = ("lnL_max", "ml_y_index", "ml_x_index", "ln_bayes", "post_x", "post_y", "x_ul")
FS_KEYS = ("lnL_max", "ml_log10_rho_index", "ln_bayes", "post_log10_rho", "log10_rho_ul")


def _user(x, y, rho2):
    """A user model with the fixed rho^2 [Ny, Nx, K]."""
    return spectra.SpectralModel(np.asarray(x, float), np.asarray(y, float), lambda f, T, xx, yy: rho2)


def _check_summaries(res, name, x, y, prefix="", kind="log-uniform", ul=0.95):
    """The reduce kernel's outputs against numpy on the device's own maps [R, Ny, Nx]."""
    r = _np(res)
    p = f"{prefix}refit_{name}_"
    ref = CO.summaries(r[p + "lnL"], x, y, kind, ul)
    assert np.array_equal(r[p + "ml_x_index"], ref["ml_log10_A_index"])
    assert np.array_equal(r[p + "ml_y_index"], ref["ml_gamma_index"])
    assert np.array_equal(r[p + "lnL_max"], ref["lnL_max"])
    np.testing.assert_allclose(r[p + "ln_bayes"], ref["ln_bayes"], rtol=1e-12, atol=1e-11)
    np.testing.assert_allclose(r[p + "post_x"], ref["post_log10_A"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r[p + "post_y"], ref["post_gamma"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r[p + "x_ul"], ref["log10_A_ul"], rtol=0, atol=1e-10)


def _xref(b, rows, name, prefix=""):
    """Extended-precision ln L [R, T] of refit model ``name`` on the device's statics, with a componentwise rounding
    bound of the projection (reduction_reference), y = V_k X_k (depth n2p), y^2, w = rho^2 / (1 + rho^2 lambda) and the
    (k, j)-ordered sum Q (depth K np), then 1/2 Q - 1/2 ldet."""
    assert RR.LONG, "the refit edge reference needs an 80-bit long double"
    st = b.compile()["fs"]
    m, arr = (st["fs"], st) if not prefix else (st["hd"]["model"], st["hd"]["arrays"])
    rf = next(r for r in st["refit"] if r["name"] == name)
    P, K, n = b.n_psr, m.n_bin, 2 * b.n_psr
    C = st["C"].cpu().numpy().reshape(b.ld, m.ncp)
    V = arr["V"].cpu().numpy().reshape(K, m.np, m.n2p)[:, :n, :n]
    lam = arr["lam"].cpu().numpy().reshape(K, m.np)[:, :n]
    r2 = rf["keep"]["rho2"].cpu().numpy().reshape(K, -1)
    ldet = rf["keep"][prefix + "ldet"].cpu().numpy()
    LD = np.longdouble
    R = rows.shape[0]
    Xh, Xl, XB = np.zeros((R, K, n)), np.zeros((R, K, n), dtype=LD), np.zeros((R, K, n))
    for a in range(P):
        h, lo, bd, _ = RR.projection(rows, C[:, :2 * K], b.toa_off[a], b.ntoa[a])
        Xh[:, :, 2 * a:2 * a + 2], Xl[:, :, 2 * a:2 * a + 2] = h.reshape(R, K, 2), lo.reshape(R, K, 2)
        XB[:, :, 2 * a:2 * a + 2] = bd.reshape(R, K, 2)
    X = Xh.astype(LD) + Xl
    y = np.einsum("kji,rki->rkj", V.astype(LD), X)
    ya = np.einsum("kji,rki->rkj", np.abs(V), np.abs(Xh))
    yb = np.einsum("kji,rki->rkj", np.abs(V), XB) + RR.gamma(m.n2p + 8) * ya
    yf = np.abs(y.astype(np.float64))
    y2b = 2 * yf * yb + yb * yb + RR.U * (yf + yb) ** 2
    w = r2[:, :, None] / (1.0 + r2[:, :, None] * lam[:, None, :])                           # [K, T, n] fp64
    wl = r2[:, :, None] / (LD(1) + r2[:, :, None] * lam[:, None, :].astype(LD))
    Q = np.einsum("rkj,ktj->rt", y * y, wl)
    QT = np.einsum("rkj,ktj->rt", (yf + yb) ** 2, w)
    QB = np.einsum("rkj,ktj->rt", y2b, w) + RR.gamma(3) * QT + RR.gamma(K * m.np + 8) * QT
    lnl = 0.5 * Q - 0.5 * ldet.astype(LD)[None]
    h, lo = RR._pair_of_ld(lnl)
    bound = 0.5 * QB + RR.U * (0.5 * QT + 0.5 * np.abs(ldet)[None] + np.abs(h))
    return dict(hi=h, lo=lo, bound=bound, terms=0.5 * QT + 0.5 * np.abs(ldet)[None])


# (K, Nx, Ny, n_psr, R, orf): K = 1 and 32, one pulsar (uncorrelated only), 2, 3, 67 and the 256-pulsar limit, T = Nx Ny
# on both sides of the 64-template block (63, 64, 65) and at the 256 x 256 limit, R = 4 and 68 (a partial second
# realization block)
EDGE_CASES = [(1, 2, 1, 1, 4, None), (32, 63, 1, 2, 68, "hd"), (14, 8, 8, 67, 4, "hd"), (32, 13, 5, 3, 68, "dipole"),
              (1, 256, 256, 2, 4, "hd"), (1, 5, 13, 256, 4, "hd"), (32, 16, 4, 67, 68, None)]


@pytest.mark.parametrize("K,Nx,Ny,P,R,orf", EDGE_CASES)
def test_refit_edges_against_extended_precision(K, Nx, Ny, P, R, orf):
    ntoas = (193,) if P == 1 else tuple((5, 6, 7, 64, 65, 193, 1025)[j % 7] for j in range(P))
    b = RR.edge_batch(ntoas, seed=400 + P + K)
    b.set_free_spectrum(log10_rho=np.linspace(-9.0, -5.0, 7), components=K, orf=orf)
    rng = np.random.default_rng(K + Nx + Ny)
    x, y = np.linspace(-1.0, 1.0, Nx), np.linspace(0.0, 1.0, Ny)
    b.set_spectral_refit({"u": _user(x, y, 10.0 ** (2 * rng.uniform(-9.0, -5.5, (Ny, Nx, K))))})
    rows = _rows(b, R, seed=K + Nx)
    res = b.free_spectrum_of(_t(b, rows), maps=True)
    keys = ()
    for prefix in ("",) + (("hd_",) if orf else ()):
        ref = _xref(b, rows, "u", prefix)
        got = res[f"{prefix}refit_u_lnL"].cpu().numpy().reshape(R, -1)
        worst, info = RR.check(got, ref, f"K={K} T={Nx * Ny} P={P} R={R} {prefix}refit lnL")
        print(f"\n[fs refit edges] K={K} T={Nx}x{Ny} P={P} R={R} {prefix or 'uncorrelated'}: |d|/bound {worst:.3f}, "
              f"|d|/(u terms) {info:.3f}")
        _check_summaries(res, "u", x, y, prefix)
        keys += tuple(f"{prefix}refit_u_{k}" for k in KEYS + ("lnL",))
    pois, _ = _poison(b, rows)
    _equal(res, b.free_spectrum_of(_t(b, pois), maps=True), keys)


def test_refit_at_grid_nodes_equals_sum_of_free_spectrum_bins():
    """A user model whose log10 rho_k(t) is the free-spectrum grid node i(t, k): the refit map is sum_k lnL[r, k, i]."""
    b, _, _ = _ng15(npsr=12)
    K, xr = 8, np.linspace(-9.0, -5.0, 41)
    b.set_free_spectrum(log10_rho=xr, components=K, orf="hd")
    rng = np.random.default_rng(7)
    Ny, Nx = 5, 24
    idx = rng.integers(0, len(xr), (Ny, Nx, K))
    b.set_spectral_refit({"nodes": _user(np.arange(Nx), np.arange(Ny), 10.0 ** (2 * xr[idx]))})
    res = _np(b.free_spectrum(128, seed=SEED, maps=True))
    kk = np.arange(K)[None, None, :]
    for prefix in ("", "hd_"):
        fs = res[prefix + "lnL"]                                                       # [R, K, NR]
        terms = fs[:, kk, idx]                                                         # [R, Ny, Nx, K]
        ref = terms.sum(axis=3)
        d = np.abs(res[f"{prefix}refit_nodes_lnL"] - ref) / (1.0 + np.abs(terms).sum(axis=3)
                                                             + 0.5 * np.abs(res[prefix + "ldet"][kk, idx]).sum(axis=2))
        print(f"\n[fs refit] {prefix or 'uncorrelated '}refit at grid nodes vs sum of fs bins: max |d| / terms = {d.max():.1e}")
        assert d.max() <= 1e-12


def test_one_bin_power_law_equals_curn_and_hd_maps():
    """At components = 1 the factorised model is exact: the power-law refit is the CURN map and the HD refit the HD map
    on the same grid and Tspan.  The grid keeps rho_1 below 10^-5.5 (inside the log10 rho range of the free spectrum's own
    tie to the one-component maps); at louder corners the two eigen forms of G^T Z G round apart further (6e-11 of the
    terms at log10 A = -13, gamma = 6)."""
    b, _, _ = _ng15(npsr=12)
    x, g = np.linspace(-16.5, -14.5, 25), np.linspace(1.0, 4.5, 11)
    b.set_free_spectrum(components=1, orf="hd")
    b.set_spectral_refit({"pl": spectra.powerlaw(x, g)})
    b.set_curn_likelihood(log10_A=x, gamma=g, components=1, Tspan=b._fs["Tspan"])
    b.set_hd_likelihood("hd")
    rows = b.generate(128, seed=SEED)
    fs = _np(b.free_spectrum_of(rows, maps=True))
    cu = _np(b.curn_likelihood_of(rows, maps=True))
    for prefix in ("", "hd_"):
        ref = cu[prefix + "lnL"]
        d = np.abs(fs[f"{prefix}refit_pl_lnL"] - ref) / (1.0 + np.abs(ref) + 0.5 * np.abs(cu[prefix + "ldet"])[None])
        print(f"\n[fs refit] one-bin {prefix or 'uncorrelated '}power-law refit vs {prefix or 'CURN '}map: "
              f"max |d| / terms = {d.max():.1e}")
        assert d.max() <= 1e-11


def test_device_matches_numpy_ng15_full():
    b, _, _ = _ng15()
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    b.set_free_spectrum(orf="hd")
    b.set_spectral_refit({"powerlaw": spectra.powerlaw(), "turnover": spectra.turnover()})
    pl = b.plan()
    pf, pr = pl["fs"], pl["fs_refit"]
    rows = b.generate(64, seed=SEED)
    res = b.free_spectrum_of(rows, maps=True)
    for name in ("powerlaw", "turnover"):
        pm = pr["models"][name]
        for prefix in ("", "hd_"):
            ref = RO.lnl_of_statics(b, pf, pm, rows.cpu().numpy(), prefix)
            got = res[f"{prefix}refit_{name}_lnL"].cpu().numpy()
            d = np.abs(got - ref) / (1.0 + np.abs(ref) + 0.5 * pm[prefix + "ldet"][None])
            print(f"\n[fs refit] {name} {prefix or 'uncorrelated '}device vs numpy, 64 realizations ng15-full: "
                  f"max |d lnL| / (1 + |lnL| + ldet/2) = {d.max():.1e}; refit statics {pr['setup_s']:.3f} s")
            assert d.max() <= 1e-11
            _check_summaries(res, name, pm["x"], pm["y"], prefix)
            assert np.array_equal(res[f"{prefix}refit_{name}_ldet"].cpu().numpy(), pm[prefix + "ldet"])
        assert np.array_equal(res[f"refit_{name}_rho2"].cpu().numpy(), pm["rho2"])
        assert np.array_equal(res[f"refit_{name}_x"].cpu().numpy(), pm["x"])
        assert np.array_equal(res[f"refit_{name}_y"].cpu().numpy(), pm["y"])


def test_device_matches_dense_oracle_small():
    b, models = _small_tm()
    b.set_free_spectrum(components=5, orf="hd")
    x = np.linspace(-15.0, -13.0, 5)
    b.set_spectral_refit({"pl": spectra.powerlaw(x, [2.0, 13 / 3, 5.0]), "to": spectra.turnover(x, [-9.0, -8.3])})
    rows = b.generate(8, seed=SEED).cpu().numpy()
    res = b.free_spectrum_of(_t(b, rows), maps=True)
    pr = b.plan()["fs_refit"]
    for name in ("pl", "to"):
        pm = pr["models"][name]
        for prefix, orf in (("", None), ("hd_", "hd")):
            ref = RO.lnl_map(b, rows, pm["rho2"].reshape(-1, 5), orf=orf, models=models).reshape(8, *pm["ldet"].shape)
            d = float(np.max(np.abs(res[f"{prefix}refit_{name}_lnL"].cpu().numpy() - ref)))
            print(f"\n[fs refit] {name} {prefix or 'uncorrelated '}device vs dense oracle, partim_small + timing model: "
                  f"max |d lnL| = {d:.1e}")
            assert d <= 1e-6


@pytest.mark.parametrize("kind,ul", [("log-uniform", 0.95), ("uniform", 0.9)])
def test_summaries_under_both_priors(kind, ul):
    b, _, _ = _ng15(npsr=12)
    b.set_free_spectrum(components=6, orf="hd")
    x, g = np.linspace(-16.0, -13.0, 40), np.linspace(0.5, 6.5, 9)
    b.set_spectral_refit({"pl": spectra.powerlaw(x, g), "to": spectra.turnover(x, [-9.2, -8.8, -8.4])},
                         amplitude_prior=kind, ul=ul)
    res = b.free_spectrum(96, seed=SEED, maps=True)
    for name, y in (("pl", g), ("to", [-9.2, -8.8, -8.4])):
        for prefix in ("", "hd_"):
            _check_summaries(res, name, x, y, prefix, kind, ul)
        import torch
        assert torch.equal(res[f"refit_{name}_ln_bayes_hd_curn"],
                           res[f"hd_refit_{name}_ln_bayes"] - res[f"refit_{name}_ln_bayes"])


def test_bit_identity_across_chunk_real0_maps_paths_and_sub_blocks():
    import torch
    b, _, _ = _ng15(npsr=12)
    b.set_free_spectrum(log10_rho=np.linspace(-9.0, -5.0, 70), components=10, orf="hd")
    R = 200
    plain = b.free_spectrum(R, seed=SEED, maps=True)                   # the free spectrum alone
    x = np.linspace(-16.0, -13.0, 33)
    b.set_spectral_refit({"pl": spectra.powerlaw(x, np.linspace(1, 6, 7)), "to": spectra.turnover(x)})
    fk = FS_KEYS + tuple("hd_" + k for k in FS_KEYS) + ("ln_bayes_hd_curn", "lnL", "hd_lnL")
    keys = tuple(f"{p}refit_{n}_{k}" for n in ("pl", "to") for p in ("", "hd_") for k in KEYS) + \
        ("refit_pl_ln_bayes_hd_curn", "refit_to_ln_bayes_hd_curn")
    mk = tuple(f"{p}refit_{n}_lnL" for n in ("pl", "to") for p in ("", "hd_"))
    a = b.free_spectrum(R, seed=SEED, maps=True)
    _equal(a, plain, fk)                                                # a refit leaves the free spectrum unchanged
    _equal(a, b.free_spectrum(R, seed=SEED, chunk=64), keys)
    c0 = b.free_spectrum(96, seed=SEED, maps=True, timers={})
    c1 = b.free_spectrum(R - 96, seed=SEED, real0=96, chunk=52, maps=True)
    for k in keys + mk:
        assert torch.equal(a[k], torch.cat([c0[k], c1[k]])), k
    rows = b.generate(R, seed=SEED)
    _equal(a, b.free_spectrum_of(rows, maps=True), keys + mk + fk)
    _equal(a, b.free_spectrum_of(rows), keys)
    per_real = 8 * 33 * 41                                             # the turnover map, the larger one
    for n_sub in (40, 128):                             # map scratch sub-blocks below and above one realization block
        b.GRID_MAP_BYTES = n_sub * per_real
        t = {}
        _equal(a, b.free_spectrum_of(rows, timers=t), keys)
        names = [e[0] for e in t["events"]]
        assert names.count("fs_y2") == 1 and names.count("hd_fs_y2") == 1
        n_refit = names.count("fs_refit")                              # the turnover map in -(-R // n_sub) sub-blocks
        assert n_refit >= -(-R // n_sub) + 1 and names.count("hd_fs_refit") == names.count("refit_reduce") == n_refit
    del b.GRID_MAP_BYTES
    for name, y in (("pl", np.linspace(1, 6, 7)), ("to", np.linspace(-9.5, -7.5, 41))):
        _check_summaries(a, name, x, y)


def test_null_mean_of_q():
    """Under the generating noise model y_kj ~ N(0, lambda_kj) in both models: Q = 2 lnL + ldet has mean
    sum_k sum_j w_kj lambda_kj (the variance is not that of independent bins: the timing model couples them)."""
    b, _, _ = _ng15(npsr=10, gwb=False)
    K = 5
    b.set_free_spectrum(components=K, orf="hd")
    x = np.array([-15.0, -14.0, -13.0])
    b.set_spectral_refit({"pl": spectra.powerlaw(x, [13 / 3])})
    pl = b.plan()
    pf, pm = pl["fs"], pl["fs_refit"]["models"]["pl"]
    res = b.free_spectrum(4096, seed=SEED, maps=True)
    r2 = pm["rho2_kt"]                                                              # [K, T]
    for prefix, lam in (("", pf["eig"].transpose(1, 0, 2).reshape(K, -1)), ("hd_", pf["hd_eig"])):
        Q = 2 * res[f"{prefix}refit_pl_lnL"].cpu().numpy().reshape(4096, -1) + pm[prefix + "ldet"].ravel()[None]
        for t in range(3):
            w = r2[:, t, None] / (1 + r2[:, t, None] * lam)
            mu = float(np.sum(w * lam))
            z = (Q[:, t].mean() - mu) / (Q[:, t].std(ddof=1) / np.sqrt(Q.shape[0]))
            print(f"\n[fs refit law] {prefix or 'uncorrelated '}H0 log10_A={x[t]}: mean {Q[:, t].mean():.4g} vs {mu:.4g} "
                  f"({z:+.2f} standard errors)")
            assert abs(z) < 5


def _injection(turnover):
    """Free spectrum (K = 10) with the power-law and turnover refits on ng15-epoch (67 pulsars, quadratic timing model),
    256 realizations of a loud ``set_gwb`` at log10 A = -14, gamma = 13/3, with a turnover at the third bin (beta = 1) or
    without; returns (outputs, log10 f0)."""
    b, _, _ = _ng15_epoch(npsr=None, gw_log10_A=-14.0)
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2)
    b.set_free_spectrum(components=10)
    lf0 = float(np.log10(3.0 / b._fs["Tspan"]))                                    # f0 at the third bin
    if turnover:
        b.set_gwb(-14.0, 13 / 3, turnover=True, f0=10.0**lf0, beta=1, power=1)
    b.set_spectral_refit({"powerlaw": spectra.powerlaw(), "turnover": spectra.turnover()})
    return _np(b.free_spectrum(256, seed=SEED)), lf0


def test_power_law_injection():
    """The loud power law is detected by both refits.  Its ML point is biased to a flatter, louder power law: the
    factorised likelihood of bin k holds no signal in the other bins, so the power that the timing model and the
    non-orthogonal basis of pulsars shorter than Tspan leak from the loud lowest bins into bin k reads as bin-k power."""
    res, _ = _injection(False)
    m = spectra.powerlaw()
    ml_a = np.median(m.x[res["refit_powerlaw_ml_x_index"]])
    ml_g = np.median(m.y[res["refit_powerlaw_ml_y_index"]])
    lb = np.median(res["refit_powerlaw_ln_bayes"])
    print(f"\n[fs refit injection] set_gwb power law log10_A = -14, gamma = 13/3, 256 realizations: median ln B "
          f"{lb:.1f}, median ML log10_A {ml_a:.3f} (margin to 0.25: {0.25 - abs(ml_a + 14):.3f}), gamma {ml_g:.3f} "
          f"(margin to 1: {1 - abs(ml_g - 13 / 3):.3f})")
    assert lb > 10 and np.median(res["refit_turnover_ln_bayes"]) > 10
    assert ml_a > -14.0 and ml_g < 13 / 3                              # the direction of the leakage bias


def test_turnover_injection_recovers_f0():
    res, lf0 = _injection(True)
    to = spectra.turnover()
    lb = np.median(res["refit_turnover_ln_bayes"] - res["refit_powerlaw_ln_bayes"])
    ml = np.median(to.y[res["refit_turnover_ml_y_index"]])
    print(f"\n[fs refit injection] set_gwb turnover log10_f0 = {lf0:.3f}: median ln B_turnover/powerlaw = {lb:.2f}, "
          f"median ML log10_f0 {ml:.3f} (margin {0.3 - abs(ml - lf0):.3f})")
    assert abs(ml - lf0) <= 0.3
