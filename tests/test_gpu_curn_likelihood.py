"""GPU tests of the CURN likelihood (``PulsarBatch.curn_likelihood`` / ``curn_likelihood_of`` -> ``ptar_os_project`` +
``ptar_curn_grid`` + ``ptar_curn_reduce``): the device against the dense oracle and against numpy on the plan's
statics, edge shapes against an extended-precision evaluation with a rounding bound, alignment slots holding NaN and
+-inf, the summaries against numpy on the device's own map, bit-identity across chunking, real0 splits, maps and
paths, the exact law of Q under the noise model and under an injected common process."""
import numpy as np
import pytest

from tests import curn_oracle as CO
from tests import reduction_reference as RR
from tests import timing_oracle as TO
from tests.test_gpu_reduction_edges import _equal, _np, _poison, _rows, _t

pytestmark = pytest.mark.gpu

SEED = 20250922
X_GRID = np.linspace(-15.5, -13.0, 6)
G_GRID = np.array([2.0, 13.0 / 3.0, 6.5])
KEYS = ("lnL_max", "ml_gamma_index", "ml_log10_A_index", "ln_bayes", "post_log10_A", "post_gamma", "log10_A_ul")


def _check_summaries(res, x, gam, kind="log-uniform", ul=0.95):
    """The reduce kernel's outputs against numpy on the device's own map: argmax and max exact, the rest to rounding."""
    r = _np(res)
    ref = CO.summaries(r["lnL"], x, gam, kind, ul)
    assert np.array_equal(r["ml_gamma_index"], ref["ml_gamma_index"])
    assert np.array_equal(r["ml_log10_A_index"], ref["ml_log10_A_index"])
    assert np.array_equal(r["lnL_max"], ref["lnL_max"])
    np.testing.assert_allclose(r["ln_bayes"], ref["ln_bayes"], rtol=1e-12, atol=1e-11)
    np.testing.assert_allclose(r["post_log10_A"], ref["post_log10_A"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r["post_gamma"], ref["post_gamma"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r["log10_A_ul"], ref["log10_A_ul"], rtol=0, atol=1e-10)


def _xref(b, rows):
    """Extended-precision ln L [R, Ng, NA] on the device's statics, with a componentwise rounding bound of the
    projection (reduction_reference), the rotation y = V X, y^2, w = A^2 / (1 + A^2 lambda) and the pulsar-ordered sum
    Q (gamma_{P ncp + 8} for any order), then 1/2 Q - 1/2 ldet."""
    assert RR.LONG, "the CURN edge reference needs an 80-bit long double"
    st = b.compile()["curn"]
    m = st["curn"]
    P, nc, ncp, NG, NA = b.n_psr, m.nc, m.ncp, m.n_gamma, m.n_amp
    C = st["C"].cpu().numpy().reshape(b.ld, ncp)
    V = st["V"].cpu().numpy().reshape(P, NG, ncp, ncp)[:, :, :nc, :nc]
    lam = st["lam"].cpu().numpy().reshape(P, NG, ncp)[:, :, :nc]
    a2, ldet = st["a2"].cpu().numpy(), st["ldet"].cpu().numpy().reshape(NG, NA)
    LD = np.longdouble
    R = rows.shape[0]
    Q = np.zeros((R, NG, NA), dtype=LD)
    QB = np.zeros((R, NG, NA))
    QT = np.zeros((R, NG, NA))
    w = (a2[None, None, :, None] / (1.0 + a2[None, None, :, None] * lam[:, :, None, :]))     # [P, NG, NA, nc] fp64
    for a in range(P):
        Xh, Xl, XB, _ = RR.projection(rows, C[:, :nc], b.toa_off[a], b.ntoa[a])
        X = Xh.astype(LD) + Xl
        y = np.einsum("gji,ri->rgj", V[a].astype(LD), X)
        ya = np.einsum("gji,ri->rgj", np.abs(V[a]), np.abs(Xh))
        yb = np.einsum("gji,ri->rgj", np.abs(V[a]), XB) + RR.gamma(nc + 8) * ya
        y2 = y * y
        yf = np.abs(y.astype(np.float64))
        y2b = 2 * yf * yb + yb * yb + RR.U * (yf + yb) ** 2
        wl = a2[None, :, None] / (LD(1) + a2[None, :, None] * lam[a][:, None, :].astype(LD))   # exact w, [NG, NA, nc]
        Q += np.einsum("rgj,gkj->rgk", y2, wl)
        QB += np.einsum("rgj,gkj->rgk", y2b, w[a]) + np.einsum("rgj,gkj->rgk", (yf + yb) ** 2, RR.gamma(3) * w[a])
        QT += np.einsum("rgj,gkj->rgk", (yf + yb) ** 2, w[a])
    QB += RR.gamma(P * ncp + 8) * QT
    lnl = 0.5 * Q - 0.5 * ldet.astype(LD)[None]
    h, l = RR._pair_of_ld(lnl)
    bound = 0.5 * QB + RR.U * (0.5 * QT + 0.5 * np.abs(ldet)[None] + np.abs(h))
    return dict(hi=h, lo=l, bound=bound, terms=0.5 * QT + 0.5 * np.abs(ldet)[None])


# (K, n_gamma, n_amp, n_psr, R): K = 1 and 16, one gamma, NA on both sides of the 64-amplitude block and the 256 limit,
# one, two and 67 pulsars, R = 4 and 68 (a partial second realization block)
EDGE_CASES = [(1, 3, 2, 2, 4), (16, 1, 63, 1, 68), (4, 2, 65, 2, 68), (14, 2, 256, 67, 4), (9, 1, 64, 3, 68),
              (16, 4, 256, 2, 68)]


@pytest.mark.parametrize("K,NG,NA,P,R", EDGE_CASES)
def test_curn_edges_against_extended_precision(K, NG, NA, P, R):
    ntoas = (193,) if P == 1 else tuple((5, 6, 7, 64, 65, 193, 1025)[j % 7] for j in range(P))
    b = RR.edge_batch(ntoas, seed=200 + P + K)
    x = np.linspace(-16.0, -12.5, NA)
    gam = np.linspace(1.5, 6.0, NG) if NG > 1 else np.array([13 / 3])
    b.set_curn_likelihood(log10_A=x, gamma=gam, components=K)
    rows = _rows(b, R, seed=K + NA)
    res = b.curn_likelihood_of(_t(b, rows), maps=True)
    ref = _xref(b, rows)
    worst, info = RR.check(res["lnL"].cpu().numpy(), ref, f"K={K} Ng={NG} NA={NA} P={P} R={R} lnL")
    print(f"\n[curn edges] K={K} Ng={NG} NA={NA} P={P} R={R}: |d|/bound {worst:.3f}, |d|/(u terms) {info:.3f}")
    _check_summaries(res, x, gam)
    pois, _ = _poison(b, rows)
    _equal(res, b.curn_likelihood_of(_t(b, pois), maps=True), KEYS + ("lnL",))


def _small_tm():
    import os

    from pta_replicator_b200 import load_from_directories, make_ideal
    from pta_replicator_b200.engine import PulsarBatch
    from tests.fixtures import GOLD
    psrs = load_from_directories(os.path.join(GOLD, "partim_small", "par"), os.path.join(GOLD, "partim_small", "tim"))
    for p in psrs:
        make_ideal(p)
    b = PulsarBatch(psrs)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.1, log10_equad=-6.5)
        b.set_ecorr(i, -6.3, coarsegrain=1.0 / 86400.0)
        b.set_red(i, -13.8 - 0.1 * i, 3.5 + 0.3 * i, components=20)
        b.set_timing_model(i, poly=2)
    models = [TO.timing_design_matrix(np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0, 2)[b.order[i]]
              for i, p in enumerate(psrs)]
    return b, models


def test_device_matches_dense_oracle_small():
    b, models = _small_tm()
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    rows = b.generate(8, seed=SEED).cpu().numpy()
    res = b.curn_likelihood_of(_t(b, rows), maps=True)
    ref = CO.lnl_map(b, rows, X_GRID, G_GRID, K=6, models=models)
    d = float(np.max(np.abs(res["lnL"].cpu().numpy() - ref)))
    print(f"\n[curn] device vs dense oracle, partim_small + timing model: max |d lnL| = {d:.1e}")
    assert d <= 1e-6
    _check_summaries(res, X_GRID, G_GRID)


def _ng15(npsr=None, **kw):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("full", npsr=npsr)
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise, **kw)
    return b, psrs, noise


def test_device_matches_numpy_ng15_full():
    b, _, _ = _ng15()
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    b.set_curn_likelihood()
    pc = b.plan()["curn"]
    rows = b.generate(64, seed=SEED)
    res = b.curn_likelihood_of(rows, maps=True)
    ref = CO.lnl_of_statics(b, pc, rows.cpu().numpy())
    got = res["lnL"].cpu().numpy()
    d = np.abs(got - ref) / (1.0 + np.abs(ref) + 0.5 * pc["ldet"][None])
    print(f"\n[curn] device vs numpy, 64 realizations ng15-full: max |d lnL| / (1 + |lnL| + ldet/2) = {d.max():.1e}, "
          f"max |d lnL| = {np.abs(got - ref).max():.1e}; host statics {pc['setup_s']:.1f} s")
    assert d.max() <= 1e-11
    _check_summaries(res, pc["log10_A"], pc["gamma"])
    assert np.array_equal(res["ldet"].cpu().numpy(), pc["ldet"]) and np.array_equal(res["lam"].cpu().numpy(), pc["eig"])


def test_bit_identity_across_chunk_real0_maps_and_paths():
    b, _, _ = _ng15(npsr=12)
    b.set_curn_likelihood(log10_A=np.linspace(-17, -12.5, 70), gamma=np.linspace(1, 6, 9), components=10)
    R = 200
    a = b.curn_likelihood(R, seed=SEED, maps=True)
    _equal(a, b.curn_likelihood(R, seed=SEED, chunk=64), KEYS)
    c0 = b.curn_likelihood(96, seed=SEED, maps=True, timers={})
    c1 = b.curn_likelihood(R - 96, seed=SEED, real0=96, chunk=52, maps=True)
    import torch
    for k in KEYS + ("lnL",):
        assert torch.equal(a[k], torch.cat([c0[k], c1[k]])), k
    rows = b.generate(R, seed=SEED)                    # no timing model: the pre-fit rows the statistic reduces
    _equal(a, b.curn_likelihood_of(rows, maps=True), KEYS + ("lnL",))
    _equal(a, b.curn_likelihood_of(rows), KEYS)
    per_real = 8 * 9 * 70
    for n_sub in (40, 128):                             # map scratch sub-blocks below and above one realization block
        b.GRID_MAP_BYTES = n_sub * per_real
        t = {}
        _equal(a, b.curn_likelihood_of(rows, timers=t), KEYS)
        assert sum(1 for e in t["events"] if e[0] == "curn_grid") == -(-R // n_sub)
    del b.GRID_MAP_BYTES
    _check_summaries(a, np.linspace(-17, -12.5, 70), np.linspace(1, 6, 9))


def _q_moments_check(Q, c, what):
    """Q [N] samples of sum_j c_j chi^2_1: sample mean and variance within 4 sigma of the exact law."""
    N = Q.size
    k2, k4 = 2 * np.sum(c**2), 48 * np.sum(c**4)
    mu = np.sum(c)
    zm = (Q.mean() - mu) / np.sqrt(k2 / N)
    zv = (Q.var(ddof=1) - k2) / np.sqrt((k4 + 2 * k2**2) / N)
    print(f"\n[curn law] {what}: mean {Q.mean():.4g} vs {mu:.4g} ({zm:+.2f} sigma), var {Q.var(ddof=1):.4g} vs "
          f"{k2:.4g} ({zv:+.2f} sigma)")
    assert abs(zm) < 4 and abs(zv) < 4


def test_null_law_of_q():
    """Under the generating noise model y_j ~ N(0, lambda_j): Q = sum w_j y_j^2 has mean sum w lambda, variance
    2 sum (w lambda)^2."""
    b, _, _ = _ng15(npsr=10, gwb=False)
    x, gam = np.array([-15.0, -14.0, -13.0]), np.array([2.0, 13 / 3, 6.0])
    b.set_curn_likelihood(log10_A=x, gamma=gam)
    pc = b.plan()["curn"]
    res = b.curn_likelihood(4096, seed=SEED, maps=True)
    Qs = 2 * res["lnL"].cpu().numpy() + pc["ldet"][None]
    for g in range(3):
        for k in range(3):
            a2 = 10.0 ** (2 * x[k])
            lam = pc["eig"][:, g, :]
            _q_moments_check(Qs[:, g, k], (a2 * lam / (1 + a2 * lam)).ravel(), f"H0 gamma={gam[g]:.2f} log10_A={x[k]}")


def test_injected_common_process():
    """A CURN injected with exactly the statistic's basis (set_red at modes k / Tspan, amplitude scaled by the pulsar's
    own span, which set_red normalises by): at the true (A*, gamma*) Q = sum A*^2 lambda_j chi^2_1; at a loud amplitude
    the median maximum-likelihood point lies within one grid step of the truth."""
    from pta_replicator_b200.engine import PulsarBatch
    from pta_replicator_b200 import synthetic
    psrs, noise = synthetic.make_ng15_like("full", npsr=10)
    ev = synthetic.ng15_recipe(PulsarBatch(psrs), noise, red=False, gwb=False)
    x, gam = np.linspace(-15.0, -12.5, 26), np.linspace(2.0, 6.0, 13)
    K = 14
    ev.set_curn_likelihood(log10_A=x, gamma=gam, components=K)
    pc = ev.plan()["curn"]
    Tspan = ev._curn["Tspan"]
    for ks, gs, R, loud in ((10, 7, 1024, False), (15, 7, 256, True)):
        inj = synthetic.ng15_recipe(PulsarBatch(psrs), noise, red=False, gwb=False)
        for i in range(inj.n_psr):
            Ta = inj.t_tdb[i].max() - inj.t_tdb[i].min()
            inj.set_red(i, x[ks] + 0.5 * np.log10(Ta / Tspan), gam[gs], modes=np.arange(1, K + 1) / Tspan)
        rows = inj.generate(R, seed=SEED + ks)
        res = ev.curn_likelihood_of(rows, maps=True)
        Q = 2 * res["lnL"].cpu().numpy()[:, gs, ks] + pc["ldet"][gs, ks]
        _q_moments_check(Q, (10.0 ** (2 * x[ks]) * pc["eig"][:, gs, :]).ravel(),
                         f"H1 A*=1e{x[ks]:.1f} gamma*={gam[gs]:.2f}")
        if loud:
            mg = np.median(res["ml_gamma_index"].cpu().numpy())
            ma = np.median(res["ml_log10_A_index"].cpu().numpy())
            print(f"[curn H1] median ML index (gamma, log10_A) = ({mg}, {ma}), truth ({gs}, {ks})")
            assert abs(mg - gs) <= 1 and abs(ma - ks) <= 1
