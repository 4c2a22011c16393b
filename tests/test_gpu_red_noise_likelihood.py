"""GPU tests of the single-pulsar red-noise likelihood (``PulsarBatch.red_noise_likelihood`` / ``red_noise_likelihood_of``
-> ``ptar_os_project`` + ``ptar_rn_grid`` + ``ptar_curn_reduce``): the device against the dense oracle and against numpy
on the plan's statics, its identity with the CURN likelihood, the exact laws of Q under the noise model and under an
injected red noise, bit-identity across chunking, sub-blocks, real0 splits, maps and paths, NaN isolation, edge shapes
against an extended-precision evaluation with a rounding bound, and ``ptar_os_project`` past 32 columns."""
import ctypes as C

import numpy as np
import pytest
from scipy.special import ndtri

from tests import reduction_reference as RR
from tests import rn_oracle as RO
from tests.test_gpu_curn_likelihood import G_GRID, KEYS, SEED, X_GRID, _ng15, _small_tm
from tests.test_gpu_reduction_edges import _equal, _np, _poison, _rows, _t

pytestmark = pytest.mark.gpu


def _check_summaries(res, x, gam, kind="log-uniform", ul=0.95):
    """The reduce kernel's outputs against numpy on the device's own maps: argmax and max exact, the rest to rounding."""
    r = _np(res)
    ref = RO.summaries(r["lnL"], x, gam, kind, ul)
    for k in ("ml_gamma_index", "ml_log10_A_index", "lnL_max"):
        assert np.array_equal(r[k], ref[k]), k
    np.testing.assert_allclose(r["ln_bayes"], ref["ln_bayes"], rtol=1e-12, atol=1e-11)
    np.testing.assert_allclose(r["post_log10_A"], ref["post_log10_A"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r["post_gamma"], ref["post_gamma"], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r["log10_A_ul"], ref["log10_A_ul"], rtol=0, atol=1e-10)


def test_device_matches_dense_oracle_small():
    b, models = _small_tm()                               # white + ECORR + red noise (20 components) + timing model
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=30)
    rows = b.generate(8, seed=SEED).cpu().numpy()
    res = b.red_noise_likelihood_of(_t(b, rows), maps=True)
    ref = RO.lnl_map(b, rows, X_GRID, G_GRID, K=30, models=models)
    d = float(np.max(np.abs(res["lnL"].cpu().numpy() - ref)))
    print(f"\n[rn] device vs dense oracle, partim_small + timing model, K = 30: max |d lnL| = {d:.1e}")
    assert d <= 1e-6
    _check_summaries(res, X_GRID, G_GRID)
    assert res["lnL_max"].shape == (8, 3) and res["post_log10_A"].shape == (8, 3, len(X_GRID))


def test_device_matches_numpy_ng15_full():
    b, _, _ = _ng15()
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    b.set_red_noise_likelihood()
    pr = b.plan()["rn"]
    rows = b.generate(8, seed=SEED)
    res = b.red_noise_likelihood_of(rows, maps=True)
    ref = RO.lnl_of_statics(b, pr, rows.cpu().numpy())
    got = res["lnL"].cpu().numpy()
    d = np.abs(got - ref) / (1.0 + np.abs(ref) + 0.5 * pr["ldet"][None])
    print(f"\n[rn] device vs numpy, 8 realizations ng15-full (K = 30, 97 x 57): max |d lnL| / (1 + |lnL| + ldet/2) = "
          f"{d.max():.1e}, max |d lnL| = {np.abs(got - ref).max():.1e}; host statics {pr['setup_s']:.1f} s")
    assert d.max() <= 1e-11
    _check_summaries(res, pr["log10_A"], pr["gamma"])
    assert np.array_equal(res["ldet"].cpu().numpy(), pr["ldet"]) and np.array_equal(res["lam"].cpu().numpy(), pr["eig"])
    assert np.array_equal(res["freqs"].cpu().numpy(), pr["freqs"])


def test_sum_over_pulsars_is_the_curn_likelihood():
    """No red noise in the recipe, Tspan = the array span and the CURN's K: the two statistics share C_a, Z_a and the
    eigen forms, so sum_a ldet[a] is CURN's ldet (the same additions in the same order) and sum_a lnL[:, a] is CURN's
    lnL to rounding."""
    import torch
    b, _, _ = _ng15(npsr=8, red=False)
    kw = dict(log10_A=np.linspace(-16, -13, 13), gamma=np.linspace(2, 6, 5), components=14)
    b.set_curn_likelihood(**kw)
    b.set_red_noise_likelihood(Tspan=b._curn["Tspan"], **kw)
    rows = b.generate(128, seed=SEED)
    c = b.curn_likelihood_of(rows, maps=True)
    r = b.red_noise_likelihood_of(rows, maps=True)
    ld = torch.zeros_like(c["ldet"])
    for a in range(b.n_psr):
        ld += r["ldet"][a]
    assert torch.equal(ld, c["ldet"])
    lnl = r["lnL"].cpu().numpy()
    d = np.abs(lnl.sum(axis=1) - c["lnL"].cpu().numpy())
    scale = np.abs(lnl).sum(axis=1) + r["ldet"].cpu().numpy().sum(axis=0)[None]
    print(f"\n[rn] sum_a lnL_a vs CURN: max |d| = {d.max():.1e}, max |d| / (sum |terms|) = {(d / scale).max():.1e}")
    assert np.all(d <= 1e-12 * scale)


def _q_moments(Q, c, what, n_checks):
    """Q [N] samples of sum_j c_j chi^2_1: sample mean and variance against the exact law.  The threshold keeps the
    chance that any of the ``n_checks`` (mean, variance) pairs of a correct kernel fails below 1e-4 (Bonferroni)."""
    z = ndtri(1 - 1e-4 / (4 * n_checks))
    N = Q.size
    k2, k4 = 2 * np.sum(c**2), 48 * np.sum(c**4)
    zm = (Q.mean() - np.sum(c)) / np.sqrt(k2 / N)
    zv = (Q.var(ddof=1) - k2) / np.sqrt((k4 + 2 * k2**2) / N)
    assert abs(zm) < z and abs(zv) < z, f"{what}: mean {zm:+.2f} sigma, variance {zv:+.2f} sigma (threshold {z:.2f})"
    return max(abs(zm), abs(zv))


def _law(b, pr, Qs, cov, tag, ks, gs):
    """Q = 2 lnL + ldet at the grid points (gs x ks) of every pulsar against sum_j c_j chi^2_1, with c the eigenvalues
    of W^1/2 cov(y) W^1/2, cov(y) = V_a(gamma) cov(X_a) V_a(gamma)^T and W = diag(w_j(A))."""
    nc = pr["nc"]
    n = b.n_psr * len(gs) * len(ks)
    worst = 0.0
    for a in range(b.n_psr):
        for g in gs:
            Vg = pr["V"][a, g, :nc, :nc]
            Sy = Vg @ cov[a] @ Vg.T
            for k in ks:
                w = np.sqrt(pr["a2"][k] / (1 + pr["a2"][k] * pr["eig"][a, g]))
                c = np.linalg.eigvalsh(w[:, None] * Sy * w[None, :])
                worst = max(worst, _q_moments(Qs[:, a, g, k], c, f"{tag} a={a} g={g} k={k}", n))
    print(f"\n[rn law] {tag}: {n} grid points, worst |z| = {worst:.2f}")


def test_null_law_of_q():
    """White + ECORR only: cov(X_a) = Z_a, y_j ~ N(0, lambda_j), Q has mean sum w lambda, variance 2 sum (w lambda)^2."""
    b, _, _ = _ng15(npsr=4, red=False, gwb=False)
    x, gam = np.array([-15.0, -14.0, -13.0]), np.array([2.0, 13 / 3, 6.0])
    b.set_red_noise_likelihood(log10_A=x, gamma=gam)
    pr = b.plan()["rn"]
    res = b.red_noise_likelihood(4096, seed=SEED, maps=True)
    Qs = 2 * res["lnL"].cpu().numpy() + pr["ldet"][None]
    _law(b, pr, Qs, pr["Z"], "H0", range(3), range(3))


def test_injected_red_noise_law_and_recovery():
    """set_red(a, log10_A*, gamma*) at its default 30 components lies in the statistic's basis: cov(X_a) = Z_a +
    Z_a phi_inj Z_a gives the exact law of Q at every checked grid point.  The posterior means of log10 A and gamma,
    averaged over the realizations, lie within one standard deviation (across realizations) of the truth."""
    from pta_replicator_b200.engine import PulsarBatch
    from pta_replicator_b200 import synthetic
    psrs, noise = synthetic.make_ng15_like("full", npsr=4)
    x, gam = np.linspace(-15.5, -12.5, 31), np.linspace(1.0, 6.0, 21)
    ks, gs = 15, 10                                                   # the truth: log10 A = -14.0, gamma = 3.5
    b = synthetic.ng15_recipe(PulsarBatch(psrs), noise, red=False, gwb=False)
    for i in range(b.n_psr):
        b.set_red(i, x[ks], gam[gs])
    b.set_red_noise_likelihood(log10_A=x, gamma=gam)
    pr = b.plan()["rn"]
    res = b.red_noise_likelihood(2048, seed=SEED + 1, maps=True)
    phi = 10.0 ** (2 * x[ks]) * pr["sp"][:, gs] ** 2                   # the injected prior, [P, nc]
    cov = pr["Z"] + np.einsum("aij,aj,ajk->aik", pr["Z"], phi, pr["Z"])
    Qs = 2 * res["lnL"].cpu().numpy() + pr["ldet"][None]
    _law(b, pr, Qs, cov, "H1", (0, ks, len(x) - 1), (0, gs, len(gam) - 1))
    r = _np(res)
    for name, grid, post, truth in (("log10_A", x, r["post_log10_A"], x[ks]), ("gamma", gam, r["post_gamma"], gam[gs])):
        pm = np.einsum("k,rak->ra", RO.CO.weights(grid) * grid, post)      # posterior mean per (realization, pulsar)
        m, s = pm.mean(axis=0), pm.std(axis=0, ddof=1)
        print(f"[rn H1] posterior mean {name}: {np.round(m, 3)} +- {np.round(s, 3)} (truth {truth})")
        assert np.all(np.abs(m - truth) <= s), name


def test_bit_identity_across_chunk_subblocks_real0_maps_and_paths():
    import torch
    b, _, _ = _ng15(npsr=12)
    x, gam = np.linspace(-17, -12.5, 70), np.linspace(1, 6, 19)
    b.set_red_noise_likelihood(log10_A=x, gamma=gam, components=20)
    R = 200
    a = b.red_noise_likelihood(R, seed=SEED, maps=True)
    _equal(a, b.red_noise_likelihood(R, seed=SEED, chunk=64), KEYS)
    c0 = b.red_noise_likelihood(96, seed=SEED, maps=True, timers={})
    c1 = b.red_noise_likelihood(R - 96, seed=SEED, real0=96, chunk=52, maps=True)
    for k in KEYS + ("lnL",):
        assert torch.equal(a[k], torch.cat([c0[k], c1[k]])), k
    rows = b.generate(R, seed=SEED)                    # no timing model: the pre-fit rows the statistic reduces
    _equal(a, b.red_noise_likelihood_of(rows, maps=True), KEYS + ("lnL",))
    per_real = 8 * b.n_psr * len(gam) * len(x)
    for n_sub in (40, 128):                             # map scratch sub-blocks below and above one realization block
        b.GRID_MAP_BYTES = n_sub * per_real
        t = {}
        _equal(a, b.red_noise_likelihood_of(rows, timers=t), KEYS)
        assert sum(1 for e in t["events"] if e[0] == "rn_grid") == -(-R // n_sub)
    del b.GRID_MAP_BYTES
    _check_summaries(a, x, gam)


def test_nan_in_one_pulsar_is_isolated():
    b, _, _ = _ng15(npsr=6)
    x, gam = np.linspace(-16, -13, 20), np.linspace(1, 6, 6)
    b.set_red_noise_likelihood(log10_A=x, gamma=gam, components=10)
    rows = b.generate(8, seed=SEED)
    clean = _np(b.red_noise_likelihood_of(rows, maps=True))
    s = b.toa_off[2]
    rows[3, s + 5] = float("nan")
    bad = _np(b.red_noise_likelihood_of(rows, maps=True))
    mask = np.ones((8, b.n_psr), dtype=bool)
    mask[3, 2] = False
    for k in KEYS + ("lnL",):
        assert np.array_equal(bad[k][mask], clean[k][mask]), k
    assert np.all(np.isnan(bad["lnL"][3, 2]))
    for k in ("lnL_max", "ln_bayes", "log10_A_ul"):
        assert np.isnan(bad[k][3, 2]), k
    assert np.all(np.isnan(bad["post_log10_A"][3, 2])) and np.all(np.isnan(bad["post_gamma"][3, 2]))
    assert bad["ml_gamma_index"][3, 2] == 0 and bad["ml_log10_A_index"][3, 2] == 0   # the first NaN of the map


def _xref(b, rows):
    """Extended-precision ln L [R, P, Ng, NA] on the device's statics, with a componentwise rounding bound of the
    projection (reduction_reference), the rotation y = V X, y^2, w = A^2 / (1 + A^2 lambda) and the sum over j
    (gamma_{ncp + 8} for any order), then 1/2 Q - 1/2 ldet."""
    assert RR.LONG, "the red-noise edge reference needs an 80-bit long double"
    st = b.compile()["rn"]
    m = st["rn"]
    P, nc, ncp, NG, NA = b.n_psr, m.nc, m.ncp, m.n_gamma, m.n_amp
    C_ = st["C"].cpu().numpy().reshape(b.ld, ncp)
    V = st["V"].cpu().numpy().reshape(P, NG, ncp, ncp)[:, :, :nc, :nc]
    lam = st["lam"].cpu().numpy().reshape(P, NG, ncp)[:, :, :nc]
    a2, ldet = st["a2"].cpu().numpy(), st["ldet"].cpu().numpy().reshape(P, NG, NA)
    LD = np.longdouble
    R = rows.shape[0]
    hi, lo = np.zeros((R, P, NG, NA)), np.zeros((R, P, NG, NA))
    bound, terms = np.zeros((R, P, NG, NA)), np.zeros((R, P, NG, NA))
    for a in range(P):
        w = a2[None, :, None] / (1.0 + a2[None, :, None] * lam[a][:, None, :])                  # [NG, NA, nc] fp64
        Xh, Xl, XB, _ = RR.projection(rows, C_[:, :nc], b.toa_off[a], b.ntoa[a])
        X = Xh.astype(LD) + Xl
        y = np.einsum("gji,ri->rgj", V[a].astype(LD), X)
        ya = np.einsum("gji,ri->rgj", np.abs(V[a]), np.abs(Xh))
        yb = np.einsum("gji,ri->rgj", np.abs(V[a]), XB) + RR.gamma(nc + 8) * ya
        yf = np.abs(y.astype(np.float64))
        y2b = 2 * yf * yb + yb * yb + RR.U * (yf + yb) ** 2
        wl = a2[None, :, None] / (LD(1) + a2[None, :, None] * lam[a][:, None, :].astype(LD))   # exact w
        Q = np.einsum("rgj,gkj->rgk", y * y, wl)
        QT = np.einsum("rgj,gkj->rgk", (yf + yb) ** 2, w)
        QB = np.einsum("rgj,gkj->rgk", y2b, w) + RR.gamma(3) * QT + RR.gamma(ncp + 8) * QT
        h, l = RR._pair_of_ld(0.5 * Q - 0.5 * ldet[a].astype(LD)[None])
        hi[:, a], lo[:, a] = h, l
        bound[:, a] = 0.5 * QB + RR.U * (0.5 * QT + 0.5 * np.abs(ldet[a])[None] + np.abs(h))
        terms[:, a] = 0.5 * QT + 0.5 * np.abs(ldet[a])[None]
    return dict(hi=hi, lo=lo, bound=bound, terms=terms)


# (K, n_gamma, n_amp, n_psr, R): every ncp / 8 instantiation (nc = 2, 16, 24, 32, 40, 48, 56, 60, 64), one gamma and a
# gamma group boundary (17), NA = 2 and 256 and both sides of the 64-amplitude block, 1, 2, 3 and 67 pulsars, R across
# the 64-row realization blocks (1, 63, 65)
EDGE_CASES = [(1, 3, 2, 2, 1), (8, 1, 256, 1, 63), (12, 2, 64, 2, 63), (16, 1, 2, 2, 65), (20, 17, 97, 3, 65),
              (24, 2, 130, 2, 4), (28, 1, 256, 2, 1), (30, 2, 65, 2, 65), (32, 1, 2, 67, 4)]


@pytest.mark.parametrize("K,NG,NA,P,R", EDGE_CASES)
def test_rn_edges_against_extended_precision(K, NG, NA, P, R):
    ntoas = (193,) if P == 1 else tuple((5, 6, 7, 64, 65, 193, 1025)[j % 7] for j in range(P))
    b = RR.edge_batch(ntoas, seed=300 + P + K)
    x = np.linspace(-16.0, -12.5, NA)
    gam = np.linspace(1.5, 6.0, NG) if NG > 1 else np.array([13 / 3])
    b.set_red_noise_likelihood(log10_A=x, gamma=gam, components=K)
    rows = _rows(b, R, seed=K + NA)
    res = b.red_noise_likelihood_of(_t(b, rows), maps=True)
    worst, info = RR.check(res["lnL"].cpu().numpy(), _xref(b, rows), f"K={K} Ng={NG} NA={NA} P={P} R={R} lnL")
    print(f"\n[rn edges] K={K} Ng={NG} NA={NA} P={P} R={R}: |d|/bound {worst:.3f}, |d|/(u terms) {info:.3f}")
    _check_summaries(res, x, gam)
    pois, _ = _poison(b, rows)
    _equal(res, b.red_noise_likelihood_of(_t(b, pois), maps=True), KEYS + ("lnL",))


@pytest.mark.parametrize("K", (20, 32))   # ncp = 40, 64
def test_wide_projection_against_extended_precision(K):
    b = RR.edge_batch((5, 64, 65, 193, 1025, 2100), seed=K)
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=K)
    st = b.compile()["rn"]
    rows = _rows(b, 65, seed=K)
    X = b._os_project(st, _t(b, rows), 65, None)[:65 * b.n_psr * st["ncp"]].view(65, b.n_psr, st["ncp"]).cpu().numpy()
    Cm = st["C"].cpu().numpy().reshape(b.ld, st["ncp"])
    for a in range(b.n_psr):
        h, l, bound, t = RR.projection(rows, Cm, b.toa_off[a], b.ntoa[a])
        RR.check(X[:, a], dict(hi=h, lo=l, bound=bound, terms=t), f"ncp={st['ncp']} pulsar {a}")


def test_projection_columns_unchanged_by_width():
    """Each column of ptar_os_project's X follows the same arithmetic at every width: X of C = [C32 | C32] at ncp 64
    equals, byte for byte in both halves, X of C32 at ncp 32 (the instantiation every existing statistic uses)."""
    import torch
    from pta_replicator_b200 import _cabi
    b = RR.edge_batch((5, 64, 65, 193, 1025, 2100), seed=7)
    b.set_red_noise_likelihood(log10_A=X_GRID, gamma=G_GRID, components=16)
    st = b.compile()["rn"]
    R, P, L = 65, b.n_psr, _cabi.lib()
    rows = _t(b, _rows(b, R, seed=7))
    C32 = st["C"].view(b.ld, 32)
    C64 = torch.cat([C32, C32], dim=1).contiguous()
    out = []
    for C_, nc in ((C32, 32), (C64, 64)):
        m = _cabi.OsModel(n_psr=P, n_tiles=st["n_tiles"], tiles=st["tiles"].data_ptr(), tile0=st["tile0"].data_ptr(),
                          n_tile=st["n_tile"].data_ptr(), C=C_.data_ptr(), nc=nc, ncp=nc)
        part = torch.empty(st["n_tiles"] * R * nc, dtype=torch.float64, device=b.device)
        X = torch.empty((R, P, nc), dtype=torch.float64, device=b.device)
        _cabi.check(L.ptar_os_project(rows.data_ptr(), b.ld, R, C.byref(m), part.data_ptr(), part.numel(), X.data_ptr(),
                                      _cabi.current_stream()), "ptar_os_project")
        out.append(X)
    assert torch.equal(out[1][..., :32], out[0]) and torch.equal(out[1][..., 32:], out[0])
    bad = _cabi.OsModel(n_psr=P, n_tiles=st["n_tiles"], tiles=st["tiles"].data_ptr(), tile0=st["tile0"].data_ptr(),
                        n_tile=st["n_tile"].data_ptr(), C=C64.data_ptr(), nc=66, ncp=72)
    assert L.ptar_os_project(rows.data_ptr(), b.ld, R, C.byref(bad), part.data_ptr(), part.numel(), X.data_ptr(),
                             _cabi.current_stream()) != 0
