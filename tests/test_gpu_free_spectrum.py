"""GPU tests of the factorised free-spectrum likelihood (``PulsarBatch.free_spectrum`` / ``free_spectrum_of`` ->
``ptar_os_project`` + ``ptar_fs_grid`` + ``ptar_curn_reduce``): edge shapes against an extended-precision evaluation
with a rounding bound and alignment slots holding NaN and +-inf, the device against the dense oracle and against numpy
on the plan's statics, every bin against the one-component CURN and HD kernels at Tspan / k, the summaries against numpy
on the device's own map, bit-identity across chunking, real0 splits, maps, paths and map sub-blocks, and the exact laws
of Q under the noise model and a single-bin injection, with a loud HD background favouring HD at the lowest bins."""
import numpy as np
import pytest

from pta_replicator_b200.engine import _powerlaw_prior
from tests import curn_oracle as CO
from tests import fs_oracle as FO
from tests import reduction_reference as RR
from tests.test_gpu_curn_likelihood import _ng15, _q_moments_check, _small_tm
from tests.test_gpu_hd_likelihood import _ng15_epoch
from tests.test_gpu_reduction_edges import _equal, _np, _poison, _rows, _t

pytestmark = pytest.mark.gpu

SEED = 20251017
KEYS = ("lnL_max", "ml_log10_rho_index", "ln_bayes", "post_log10_rho", "log10_rho_ul")


def _check_summaries(res, x, prefix=""):
    """The reduce kernel's outputs against numpy on the device's own maps [R, K, NR]."""
    r = _np(res)
    R, K, NR = r[prefix + "lnL"].shape
    ref = CO.summaries(r[prefix + "lnL"].reshape(R * K, 1, NR), x, [0.0])
    assert np.array_equal(r[prefix + "ml_log10_rho_index"].ravel(), ref["ml_log10_A_index"])
    assert np.array_equal(r[prefix + "lnL_max"].ravel(), ref["lnL_max"])
    np.testing.assert_allclose(r[prefix + "ln_bayes"].ravel(), ref["ln_bayes"], rtol=1e-12, atol=1e-11)
    np.testing.assert_allclose(r[prefix + "post_log10_rho"].reshape(R * K, NR), ref["post_log10_A"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r[prefix + "log10_rho_ul"].ravel(), ref["log10_A_ul"], rtol=0, atol=1e-10)
    assert not any(k.endswith(("ml_gamma_index", "post_gamma")) for k in res)


def _xref(b, rows, prefix=""):
    """Extended-precision ln L [R, K, NR] on the device's statics, with a componentwise rounding bound of the
    projection (reduction_reference), the gathered rotation y = V_k X_k (depth n2p), y^2, w = rho^2 / (1 + rho^2 lambda)
    and the j-ordered sum Q (depth np), then 1/2 Q - 1/2 ldet."""
    assert RR.LONG, "the free-spectrum edge reference needs an 80-bit long double"
    st = b.compile()["fs"]
    m, arr = (st["fs"], st) if not prefix else (st["hd"]["model"], st["hd"]["arrays"])
    P, K, NA, n = b.n_psr, m.n_bin, m.n_amp, 2 * b.n_psr
    C = st["C"].cpu().numpy().reshape(b.ld, m.ncp)
    V = arr["V"].cpu().numpy().reshape(K, m.np, m.n2p)[:, :n, :n]
    lam = arr["lam"].cpu().numpy().reshape(K, m.np)[:, :n]
    a2, ldet = st["a2"].cpu().numpy(), arr["ldet"].cpu().numpy().reshape(K, NA)
    LD = np.longdouble
    R = rows.shape[0]
    Xh, Xl, XB = (np.zeros((R, K, n)) for _ in range(3))
    Xl = Xl.astype(LD)
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
    w = a2[None, :, None] / (1.0 + a2[None, :, None] * lam[:, None, :])                      # [K, NA, n] fp64
    wl = a2[None, :, None] / (LD(1) + a2[None, :, None] * lam[:, None, :].astype(LD))
    Q = np.einsum("rkj,kij->rki", y * y, wl)
    QT = np.einsum("rkj,kij->rki", (yf + yb) ** 2, w)
    QB = np.einsum("rkj,kij->rki", y2b, w) + RR.gamma(3) * QT + RR.gamma(m.np + 8) * QT
    lnl = 0.5 * Q - 0.5 * ldet.astype(LD)[None]
    h, lo = RR._pair_of_ld(lnl)
    bound = 0.5 * QB + RR.U * (0.5 * QT + 0.5 * np.abs(ldet)[None] + np.abs(h))
    return dict(hi=h, lo=lo, bound=bound, terms=0.5 * QT + 0.5 * np.abs(ldet)[None])


# (K, NR, n_psr, R, orf): K = 1 and 32, one pulsar (uncorrelated only), 2, 3, 67 and the 256-pulsar limit, NR on both
# sides of the 64-amplitude block and the 256 limit, R = 4 and 68 (a partial second realization block)
EDGE_CASES = [(1, 2, 1, 4, None), (32, 63, 2, 68, "hd"), (14, 65, 67, 4, "hd"), (32, 64, 3, 68, "dipole"),
              (1, 256, 256, 4, "hd"), (5, 256, 67, 68, None)]


@pytest.mark.parametrize("K,NR,P,R,orf", EDGE_CASES)
def test_fs_edges_against_extended_precision(K, NR, P, R, orf):
    ntoas = (193,) if P == 1 else tuple((5, 6, 7, 64, 65, 193, 1025)[j % 7] for j in range(P))
    b = RR.edge_batch(ntoas, seed=300 + P + K)
    x = np.linspace(-9.0, -5.0, NR)
    b.set_free_spectrum(log10_rho=x, components=K, orf=orf)
    rows = _rows(b, R, seed=K + NR)
    res = b.free_spectrum_of(_t(b, rows), maps=True)
    keys = KEYS + ("lnL",)
    for prefix in ("",) + (("hd_",) if orf else ()):
        ref = _xref(b, rows, prefix)
        worst, info = RR.check(res[prefix + "lnL"].cpu().numpy(), ref, f"K={K} NR={NR} P={P} R={R} {prefix}lnL")
        print(f"\n[fs edges] K={K} NR={NR} P={P} R={R} {prefix or 'uncorrelated'}: |d|/bound {worst:.3f}, "
              f"|d|/(u terms) {info:.3f}")
        _check_summaries(res, x, prefix)
        keys += tuple(prefix + k for k in KEYS + ("lnL",))
    pois, _ = _poison(b, rows)
    _equal(res, b.free_spectrum_of(_t(b, pois), maps=True), keys)


def test_device_matches_dense_oracle_small():
    b, models = _small_tm()
    x = np.linspace(-8.5, -5.5, 7)
    b.set_free_spectrum(log10_rho=x, components=6, orf="hd")
    rows = b.generate(8, seed=SEED).cpu().numpy()
    res = b.free_spectrum_of(_t(b, rows), maps=True)
    for prefix, orf in (("", None), ("hd_", "hd")):
        ref = FO.lnl_map(b, rows, x, 6, orf=orf, models=models)
        d = float(np.max(np.abs(res[prefix + "lnL"].cpu().numpy() - ref)))
        print(f"\n[fs] {prefix or 'uncorrelated '}device vs dense oracle, partim_small + timing model: max |d lnL| = {d:.1e}")
        assert d <= 1e-6
        _check_summaries(res, x, prefix)


def test_device_matches_numpy_ng15_full():
    b, _, _ = _ng15()
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    b.set_free_spectrum(orf="hd", log10_A_common=-14.5)
    pf = b.plan()["fs"]
    rows = b.generate(64, seed=SEED)
    res = b.free_spectrum_of(rows, maps=True)
    for prefix in ("", "hd_"):
        ref = FO.lnl_of_statics(b, pf, rows.cpu().numpy(), prefix)
        got = res[prefix + "lnL"].cpu().numpy()
        d = np.abs(got - ref) / (1.0 + np.abs(ref) + 0.5 * pf[prefix + "ldet"][None])
        print(f"\n[fs] {prefix or 'uncorrelated '}device vs numpy, 64 realizations ng15-full: max |d lnL| / (1 + |lnL| + "
              f"ldet/2) = {d.max():.1e}; host statics {pf['setup_s']:.2f} s")
        assert d.max() <= 1e-11
        _check_summaries(res, pf["log10_A"], prefix)
    assert np.array_equal(res["ldet"].cpu().numpy(), pf["ldet"]) and np.array_equal(res["lam"].cpu().numpy(), pf["eig"])
    assert np.array_equal(res["hd_ldet"].cpu().numpy(), pf["hd_ldet"])
    assert np.array_equal(res["log10_rho"].cpu().numpy(), pf["log10_A"]) and res["freqs"].shape == (14,)


def test_bins_equal_shifted_one_component_curn_and_hd_maps():
    """Bin k's maps are the CURN and HD maps of components=1, Tspan = T / k, after the shift log10 A = log10 rho -
    1/2 log10 phi~_k: the new kernel against two tested kernels."""
    b, _, _ = _ng15(npsr=12)
    K, g = 6, 13 / 3
    x = np.linspace(-8.5, -5.5, 31)
    b.set_free_spectrum(log10_rho=x, components=K, orf="hd")
    rows = b.generate(128, seed=SEED)
    fs = _np(b.free_spectrum_of(rows, maps=True))
    T = b._fs["Tspan"]
    worst = 0.0
    for k in (1, 2, K):
        pt = _powerlaw_prior([k / T], g, T / k)[0]
        b.set_curn_likelihood(log10_A=x - 0.5 * np.log10(pt), gamma=[g], components=1, Tspan=T / k)
        b.set_hd_likelihood("hd")
        cu = _np(b.curn_likelihood_of(rows, maps=True))
        for prefix in ("", "hd_"):
            ref = cu[prefix + "lnL"][:, 0]
            got = fs[prefix + "lnL"][:, k - 1]
            d = np.abs(got - ref) / (1.0 + np.abs(ref) + 0.5 * np.abs(cu[prefix + "ldet"][0])[None])
            worst = max(worst, float(d.max()))
    print(f"\n[fs] bins vs one-component CURN / HD maps: max |d| / terms = {worst:.1e}")
    assert worst <= 1e-11


def test_bit_identity_across_chunk_real0_maps_paths_and_sub_blocks():
    b, _, _ = _ng15(npsr=12)
    x = np.linspace(-9.0, -5.0, 70)
    b.set_free_spectrum(log10_rho=x, components=10, orf="hd", log10_A_common=-14.3)
    keys = KEYS + tuple("hd_" + k for k in KEYS) + ("ln_bayes_hd_curn",)
    R = 200
    a = b.free_spectrum(R, seed=SEED, maps=True)
    _equal(a, b.free_spectrum(R, seed=SEED, chunk=64), keys)
    c0 = b.free_spectrum(96, seed=SEED, maps=True, timers={})
    c1 = b.free_spectrum(R - 96, seed=SEED, real0=96, chunk=52, maps=True)
    import torch
    for k in keys + ("lnL", "hd_lnL"):
        assert torch.equal(a[k], torch.cat([c0[k], c1[k]])), k
    rows = b.generate(R, seed=SEED)
    _equal(a, b.free_spectrum_of(rows, maps=True), keys + ("lnL", "hd_lnL"))
    _equal(a, b.free_spectrum_of(rows), keys)
    per_real = 8 * 10 * 70
    for n_sub in (40, 128):                             # map scratch sub-blocks below and above one realization block
        b.GRID_MAP_BYTES = n_sub * per_real
        t = {}
        _equal(a, b.free_spectrum_of(rows, timers=t), keys)
        assert sum(1 for e in t["events"] if e[0] == "fs_grid") == -(-R // n_sub)
        assert sum(1 for e in t["events"] if e[0] == "hd_fs_grid") == -(-R // n_sub)
    del b.GRID_MAP_BYTES
    assert torch.equal(a["ln_bayes_hd_curn"], a["hd_ln_bayes"] - a["ln_bayes"])
    _check_summaries(a, x)
    _check_summaries(a, x, "hd_")


def test_null_law_of_q():
    """Under the generating noise model y_j ~ N(0, lambda_j) in both models: Q = 2 lnL + ldet has the law of
    sum_j w_j lambda_j chi^2_1."""
    b, _, _ = _ng15(npsr=10, gwb=False)
    x = np.array([-7.5, -6.5, -5.5])
    b.set_free_spectrum(log10_rho=x, components=5, orf="hd")
    pf = b.plan()["fs"]
    res = b.free_spectrum(4096, seed=SEED, maps=True)
    for prefix, lam in (("", pf["eig"].transpose(1, 0, 2).reshape(5, -1)), ("hd_", pf["hd_eig"])):
        Qs = 2 * res[prefix + "lnL"].cpu().numpy() + pf[prefix + "ldet"][None]
        for k in (0, 4):
            for i in range(3):
                a2 = 10.0 ** (2 * x[i])
                _q_moments_check(Qs[:, k, i], a2 * lam[k] / (1 + a2 * lam[k]), f"fs {prefix}H0 bin {k + 1} log10_rho={x[i]}")


def test_single_bin_injection():
    """A red process in bin k alone (set_red at the mode k / Tspan, amplitude scaled by the pulsar's own span, which
    set_red normalises by): at the true rho, Q = sum rho*^2 lambda_j chi^2_1; loud, the median ML lies within one grid
    step of the truth."""
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("full", npsr=10)
    ev = synthetic.ng15_recipe(PulsarBatch(psrs), noise, red=False, gwb=False)
    x = np.linspace(-8.0, -5.0, 31)
    K, g = 8, 13 / 3
    ev.set_free_spectrum(log10_rho=x, components=K)
    pf = ev.plan()["fs"]
    T = ev._fs["Tspan"]
    for kb, ir, R, loud in ((3, 10, 1024, False), (3, 22, 256, True)):
        inj = synthetic.ng15_recipe(PulsarBatch(psrs), noise, red=False, gwb=False)
        pt = _powerlaw_prior([kb / T], g, T)[0]
        for i in range(inj.n_psr):
            Ta = inj.t_tdb[i].max() - inj.t_tdb[i].min()
            inj.set_red(i, x[ir] - 0.5 * np.log10(pt) + 0.5 * np.log10(Ta / T), g, modes=np.array([kb / T]))
        res = ev.free_spectrum_of(inj.generate(R, seed=SEED + ir), maps=True)
        Q = 2 * res["lnL"].cpu().numpy()[:, kb - 1, ir] + pf["ldet"][kb - 1, ir]
        _q_moments_check(Q, 10.0 ** (2 * x[ir]) * pf["eig"][:, kb - 1].ravel(), f"fs H1 bin {kb} log10_rho*={x[ir]:.1f}")
        if loud:
            ml = np.median(res["ml_log10_rho_index"].cpu().numpy()[:, kb - 1])
            print(f"[fs H1] median ML index {ml}, truth {ir}")
            assert abs(ml - ir) <= 1


def test_recipe_gwb_injection_favours_hd_at_low_bins():
    """A loud HD GWB of ``set_gwb`` (67 ng15-epoch pulsars, spin-down quadratic marginalised): the median
    ln B_HD/CURN of the lowest bins is positive."""
    b, _, _ = _ng15_epoch(npsr=None, gw_log10_A=-14.0)
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2)
    b.set_free_spectrum(log10_rho=np.linspace(-9.0, -5.0, 41), components=5, orf="hd")
    res = b.free_spectrum(256, seed=SEED)
    lb = res["ln_bayes_hd_curn"].cpu().numpy()
    med = np.median(lb, axis=0)
    print(f"\n[fs recipe] set_gwb HD at log10_A = -14.0, {b.n_psr} pulsars, 256 realizations: median ln B_HD/CURN per "
          f"bin = {' / '.join(f'{v:.2f}' for v in med)}")
    assert med[0] > 0 and med[1] > 0
