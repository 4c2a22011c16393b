"""GPU tests of the HD likelihood (``PulsarBatch.set_hd_likelihood`` -> ``ptar_hd_grid`` + ``ptar_curn_reduce`` on the HD
map): the device against the dense stacked-covariance oracle and against numpy on the plan's statics, edge shapes
against an extended-precision evaluation with a rounding bound, alignment slots holding NaN and +-inf, the summaries
against numpy on the device's own map, bit-identity across chunking, real0 splits, maps and paths, CURN outputs
unchanged by the registration, the exact law of Q under the noise model and under an HD process injected in the
statistic's basis, and the HD-vs-CURN Bayes factor of loud injections."""
import numpy as np
import pytest

from tests import curn_oracle as CO
from tests import hd_oracle as HO
from tests import os_oracle as OO
from tests import reduction_reference as RR
from tests.test_gpu_curn_likelihood import KEYS, _check_summaries, _ng15, _q_moments_check, _small_tm
from tests.test_gpu_reduction_edges import _equal, _np, _poison, _rows, _t

pytestmark = pytest.mark.gpu

SEED = 20251016
X_GRID = np.linspace(-15.5, -13.0, 6)
G_GRID = np.array([2.0, 13.0 / 3.0, 6.5])
HD_KEYS = tuple("hd_" + k for k in KEYS) + ("ln_bayes_hd_curn",)


def _hd_view(res):
    """The HD outputs under the CURN names, for the summary checks."""
    out = {k: res["hd_" + k] for k in KEYS}
    if "hd_lnL" in res:
        out["lnL"] = res["hd_lnL"]
    return out


def _check_bayes(res):
    import torch
    assert torch.equal(res["ln_bayes_hd_curn"], res["hd_ln_bayes"] - res["ln_bayes"])


def _xref(b, rows):
    """Extended-precision HD ln L [R, Ng, NA] on the device's statics, with a componentwise rounding bound of the
    projection (reduction_reference), the rotation y = V X over the stacked axis (gamma_{P ncp + 8}), y^2,
    w = A^2 / (1 + A^2 lambda) and the j-ordered sum Q (gamma_{N + 8} for any order), then 1/2 Q - 1/2 ldet."""
    assert RR.LONG, "the HD edge reference needs an 80-bit long double"
    st = b.compile()["curn"]
    m, hm = st["curn"], st["hd"]["model"]
    P, nc, ncp, NG, NA, N, NP = b.n_psr, m.nc, m.ncp, m.n_gamma, m.n_amp, hm.n, hm.np
    C = st["C"].cpu().numpy().reshape(b.ld, ncp)
    arr = st["hd"]["arrays"]
    V = arr["V"].cpu().numpy().reshape(NG, NP, P * ncp)[:, :N]
    lam = arr["lam"].cpu().numpy().reshape(NG, NP)[:, :N]
    a2, ldet = st["a2"].cpu().numpy(), arr["ldet"].cpu().numpy().reshape(NG, NA)
    LD = np.longdouble
    R = rows.shape[0]
    Xh, Xl, XB = (np.zeros((R, P * ncp)) for _ in range(3))
    for a in range(P):
        h, l, bnd, _ = RR.projection(rows, C[:, :nc], b.toa_off[a], b.ntoa[a])
        Xh[:, a * ncp:a * ncp + nc], Xl[:, a * ncp:a * ncp + nc], XB[:, a * ncp:a * ncp + nc] = h, l, bnd
    X = Xh.astype(LD) + Xl
    y = np.einsum("gjk,rk->rgj", V.astype(LD), X)
    ya = np.einsum("gjk,rk->rgj", np.abs(V), np.abs(Xh))
    yb = np.einsum("gjk,rk->rgj", np.abs(V), XB) + RR.gamma(P * ncp + 8) * ya
    yf = np.abs(y.astype(np.float64))
    y2b = 2 * yf * yb + yb * yb + RR.U * (yf + yb) ** 2
    w = a2[None, :, None] / (1.0 + a2[None, :, None] * lam[:, None, :])                 # [NG, NA, N] fp64
    wl = a2[None, :, None] / (LD(1) + a2[None, :, None] * lam[:, None, :].astype(LD))    # exact w
    Q = np.einsum("rgj,gkj->rgk", y * y, wl)
    QT = np.einsum("rgj,gkj->rgk", (yf + yb) ** 2, w)
    QB = np.einsum("rgj,gkj->rgk", y2b, w) + RR.gamma(3) * QT + RR.gamma(N + 8) * QT
    lnl = 0.5 * Q - 0.5 * ldet.astype(LD)[None]
    h, l = RR._pair_of_ld(lnl)
    bound = 0.5 * QB + RR.U * (0.5 * QT + 0.5 * np.abs(ldet)[None] + np.abs(h))
    return dict(hi=h, lo=l, bound=bound, terms=0.5 * QT + 0.5 * np.abs(ldet)[None])


# (K, n_gamma, n_amp, n_psr, R, orf): K = 1, 4, 16; N = n_psr 2K off the 32-row block (4, 24, 54, 670, 1876) and on it
# (64, 96); NA on both sides of the 64 and 128 amplitude widths and at the 256 limit; 1..4 gammas; 2, 3 and 67 pulsars;
# R = 1, 4, 65, 130 (partial and several realization blocks); the HD template and a matrix whose diagonal is not 1
EDGE_CASES = [(1, 3, 2, 2, 4, "hd"), (16, 1, 63, 2, 65, "hd"), (4, 2, 65, 3, 130, "psd"), (14, 2, 256, 67, 4, "hd"),
              (9, 4, 64, 3, 1, "dipole"), (16, 4, 256, 3, 130, "psd"), (5, 1, 128, 67, 65, "hd"),
              (4, 3, 129, 2, 65, "monopole")]


@pytest.mark.parametrize("K,NG,NA,P,R,orf", EDGE_CASES)
def test_hd_edges_against_extended_precision(K, NG, NA, P, R, orf):
    ntoas = tuple((5, 6, 7, 64, 65, 193, 1025)[j % 7] for j in range(P))
    b = RR.edge_batch(ntoas, seed=300 + P + K)
    x = np.linspace(-16.0, -12.5, NA)
    gam = np.linspace(1.5, 6.0, NG) if NG > 1 else np.array([13 / 3])
    b.set_curn_likelihood(log10_A=x, gamma=gam, components=K)
    if orf == "psd":
        A = np.random.default_rng(P + K).standard_normal((P, P))
        orf = A @ A.T / P
    b.set_hd_likelihood(orf=orf)
    rows = _rows(b, R, seed=K + NA)
    res = b.curn_likelihood_of(_t(b, rows), maps=True)
    ref = _xref(b, rows)
    worst, info = RR.check(res["hd_lnL"].cpu().numpy(), ref, f"K={K} Ng={NG} NA={NA} P={P} R={R} hd_lnL")
    print(f"\n[hd edges] K={K} Ng={NG} NA={NA} P={P} R={R} N={P * 2 * K}: |d|/bound {worst:.3f}, "
          f"|d|/(u terms) {info:.3f}")
    _check_summaries(_hd_view(res), x, gam)
    _check_bayes(res)
    pois, _ = _poison(b, rows)
    _equal(res, b.curn_likelihood_of(_t(b, pois), maps=True), KEYS + HD_KEYS + ("lnL", "hd_lnL"))


def test_device_matches_dense_oracle_small():
    b, models = _small_tm()
    b.set_curn_likelihood(log10_A=X_GRID, gamma=G_GRID, components=6)
    b.set_hd_likelihood()
    rows = b.generate(8, seed=SEED).cpu().numpy()
    res = b.curn_likelihood_of(_t(b, rows), maps=True)
    ref, ld = HO.lnl_map(b, rows, X_GRID, G_GRID, K=6, models=models)
    d = float(np.max(np.abs(res["hd_lnL"].cpu().numpy() - ref)))
    dl = float(np.max(np.abs(res["hd_ldet"].cpu().numpy() - ld) / np.maximum(1.0, np.abs(ld))))
    print(f"\n[hd] device vs dense oracle, partim_small + timing model: max |d lnL| = {d:.1e}, ldet rel {dl:.1e}")
    assert d <= 1e-6 and dl <= 1e-9
    _check_summaries(_hd_view(res), X_GRID, G_GRID)
    _check_bayes(res)


def test_device_matches_numpy_ng15_full():
    b, _, _ = _ng15()
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    gam = np.array([2.0, 13.0 / 3.0, 6.0])
    b.set_curn_likelihood(gamma=gam)
    b.set_hd_likelihood()
    pl = b.plan()
    pc, ph = pl["curn"], pl["hd"]
    rows = b.generate(64, seed=SEED)
    res = b.curn_likelihood_of(rows, maps=True)
    ref = HO.lnl_of_statics(b, pc, ph, rows.cpu().numpy())
    got = res["hd_lnL"].cpu().numpy()
    d = np.abs(got - ref) / (1.0 + np.abs(ref) + 0.5 * ph["ldet"][None])
    lb = res["ln_bayes_hd_curn"].cpu().numpy()
    print(f"\n[hd] device vs numpy, 64 realizations ng15-full (N = {ph['n']}): max |d lnL| / (1 + |lnL| + ldet/2) = "
          f"{d.max():.1e}, max |d lnL| = {np.abs(got - ref).max():.1e}; host statics {ph['setup_s']:.1f} s for "
          f"{len(gam)} gammas, V {ph['nbytes'] / 1e6:.0f} MB; ln B_HD/CURN median {np.median(lb):.2f}")
    assert d.max() <= 1e-11
    _check_summaries(_hd_view(res), pc["log10_A"], gam)
    _check_bayes(res)
    assert np.array_equal(res["hd_ldet"].cpu().numpy(), ph["ldet"]) and np.array_equal(res["hd_lam"].cpu().numpy(),
                                                                                      ph["eig"])


def test_bit_identity_across_chunk_real0_maps_and_paths():
    import torch
    b, _, _ = _ng15(npsr=12)
    x, gam = np.linspace(-17, -12.5, 70), np.linspace(1, 6, 9)
    b.set_curn_likelihood(log10_A=x, gamma=gam, components=10)
    R = 200
    plain = b.curn_likelihood(R, seed=SEED, maps=True)
    assert not any(k.startswith("hd_") for k in plain)
    b.set_hd_likelihood()
    timers = {}
    a = b.curn_likelihood(R, seed=SEED, maps=True, timers=timers)
    names = {n for n, _, _ in timers["events"]}
    assert {"curn_grid", "curn_reduce", "hd_grid", "hd_reduce"} <= names
    _equal(a, plain, KEYS + ("lnL", "ldet", "lam"))       # the CURN outputs do not see the HD registration
    _equal(a, b.curn_likelihood(R, seed=SEED, chunk=64), KEYS + HD_KEYS)
    c0 = b.curn_likelihood(96, seed=SEED, maps=True)
    c1 = b.curn_likelihood(R - 96, seed=SEED, real0=96, chunk=52, maps=True)
    for k in KEYS + HD_KEYS + ("lnL", "hd_lnL"):
        assert torch.equal(a[k], torch.cat([c0[k], c1[k]])), k
    rows = b.generate(R, seed=SEED)
    _equal(a, b.curn_likelihood_of(rows, maps=True), KEYS + HD_KEYS + ("lnL", "hd_lnL"))
    _equal(a, b.curn_likelihood_of(rows), KEYS + HD_KEYS)
    per_real = 8 * len(gam) * len(x)
    for n_sub in (40, 128):                             # map scratch sub-blocks below and above one realization block
        b.GRID_MAP_BYTES = n_sub * per_real
        t = {}
        _equal(a, b.curn_likelihood_of(rows, timers=t), KEYS + HD_KEYS)
        for name in ("curn_grid", "hd_grid"):
            assert sum(1 for e in t["events"] if e[0] == name) == -(-R // n_sub), name
    del b.GRID_MAP_BYTES
    _check_summaries(_hd_view(a), x, gam)
    _check_bayes(a)


def test_null_law_of_q():
    """Under the generating noise model y_j ~ N(0, lambda_j): Q = sum w_j y_j^2 has mean sum w lambda, variance
    2 sum (w lambda)^2."""
    b, _, _ = _ng15(npsr=10, gwb=False)
    x, gam = np.array([-15.0, -14.0, -13.0]), np.array([2.0, 13 / 3, 6.0])
    b.set_curn_likelihood(log10_A=x, gamma=gam)
    b.set_hd_likelihood()
    ph = b.plan()["hd"]
    res = b.curn_likelihood(4096, seed=SEED, maps=True)
    Qs = 2 * res["hd_lnL"].cpu().numpy() + ph["ldet"][None]
    for g in range(3):
        for k in range(3):
            a2 = 10.0 ** (2 * x[k])
            lam = ph["eig"][g]
            _q_moments_check(Qs[:, g, k], a2 * lam / (1 + a2 * lam), f"HD H0 gamma={gam[g]:.2f} log10_A={x[k]}")


def _inject_hd(b, rows, log10_A, gamma, K, Tspan, seed):
    """rows + F_a c_a, c ~ N(0, A^2 Gamma_HD (x) phi~(gamma)) drawn on the host in the statistic's own basis."""
    Gam = HO.orf_matrix(b, "hd")
    mu, E = np.linalg.eigh(Gam)
    Bm = E * np.sqrt(np.maximum(mu, 0.0))
    sp = np.sqrt(OO.phi_tilde(K, gamma, Tspan))
    z = np.random.default_rng(seed).standard_normal((rows.shape[0], b.n_psr, 2 * K))
    c = 10.0 ** log10_A * np.einsum("ab,rbi->rai", Bm, z) * sp[None, None, :]
    out = rows.copy()
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        out[:, s:s + n] += c[:, i] @ OO.gw_basis(b.t_tdb[i], K, Tspan).T
    return out


def test_injected_hd_process():
    """An HD process injected exactly in the statistic's basis: at the true (A*, gamma*) Q = sum A*^2 lambda_j chi^2_1;
    at a loud amplitude the median maximum-likelihood point lies within one grid step of the truth and the median
    ln B_HD/CURN is positive."""
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("full", npsr=10)
    b = synthetic.ng15_recipe(PulsarBatch(psrs), noise, red=False, gwb=False)
    x, gam = np.linspace(-15.0, -12.5, 26), np.linspace(2.0, 6.0, 13)
    K = 14
    b.set_curn_likelihood(log10_A=x, gamma=gam, components=K)
    b.set_hd_likelihood()
    ph = b.plan()["hd"]
    Tspan = b._curn["Tspan"]
    for ks, gs, R, loud in ((10, 7, 1024, False), (15, 7, 256, True)):
        rows = _inject_hd(b, b.generate(R, seed=SEED + ks).cpu().numpy(), x[ks], gam[gs], K, Tspan, seed=ks)
        res = b.curn_likelihood_of(_t(b, rows), maps=True)
        Q = 2 * res["hd_lnL"].cpu().numpy()[:, gs, ks] + ph["ldet"][gs, ks]
        _q_moments_check(Q, 10.0 ** (2 * x[ks]) * ph["eig"][gs], f"HD H1 A*=1e{x[ks]:.1f} gamma*={gam[gs]:.2f}")
        if loud:
            mg = np.median(res["hd_ml_gamma_index"].cpu().numpy())
            ma = np.median(res["hd_ml_log10_A_index"].cpu().numpy())
            lb = res["ln_bayes_hd_curn"].cpu().numpy()
            print(f"[hd H1] median ML index (gamma, log10_A) = ({mg}, {ma}), truth ({gs}, {ks}); ln B_HD/CURN "
                  f"median {np.median(lb):.2f}, 10/90 % {np.percentile(lb, 10):.2f} / {np.percentile(lb, 90):.2f}")
            assert abs(mg - gs) <= 1 and abs(ma - ks) <= 1 and np.median(lb) > 0


def test_recipe_gwb_injection_favours_hd():
    """The product's own injection path: a loud HD GWB of ``set_gwb`` (67 ng15-epoch pulsars, spin-down quadratic
    marginalised, which absorbs the injection's power below 1 / Tspan) gives a positive median ln B_HD/CURN."""
    b, _, _ = _ng15_epoch(npsr=None, gw_log10_A=-14.0)
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2)
    b.set_curn_likelihood(log10_A=np.linspace(-16.0, -13.0, 31), gamma=[13 / 3])
    b.set_hd_likelihood()
    res = b.curn_likelihood(256, seed=SEED)
    lb = res["ln_bayes_hd_curn"].cpu().numpy()
    q = np.percentile(lb, [5, 25, 50, 75, 95])
    print(f"\n[hd recipe] set_gwb HD at log10_A = -14.0, {b.n_psr} ng15-epoch pulsars, 256 realizations: ln B_HD/CURN "
          f"5/25/50/75/95 % = {' / '.join(f'{v:.2f}' for v in q)}; P(ln B > 0) = {np.mean(lb > 0):.2f}; median "
          f"ML log10_A = {np.median(res['hd_ml_log10_A_index'].cpu().numpy()) * 0.1 - 16.0:.1f}")
    assert np.median(lb) > 0


def _ng15_epoch(npsr, **kw):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("epoch", npsr=npsr)
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise, **kw)
    return b, psrs, noise
