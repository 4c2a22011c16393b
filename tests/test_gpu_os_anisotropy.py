"""GPU tests of the anisotropy statistics of the optimal statistic (``PulsarBatch.set_os_anisotropy`` ->
``ptar_os_aniso``): the device against the plan's statics applied in numpy, existing outputs unchanged by the
registration, bit-identity across chunking, real0 splits and paths, the exact laws under the noise model, the
injected-signal means (in the statistic's own basis and from ``set_gwb(lmax=6)`` against the dense oracle's exact
expectation) and an edge sweep against the extended-precision reference of tests/reduction_reference.py."""
import numpy as np
import pytest

from tests import aniso_oracle as AO
from tests import os_oracle as OO
from tests import reduction_reference as RR
from tests import timing_oracle as TO
from tests.test_gpu_optimal_statistic import SEED, _batch, _ng15

pytestmark = pytest.mark.gpu

ANISO_KEYS = ("clm", "aniso_z", "aniso_chi2", "radio_snr_max", "radio_argmax", "radio_snr")


def _pair_d(b, po, rows):
    """d [R, n_pairs] = x_a . x_b of host rows, with the plan's C."""
    nc = po["nc"]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :nc]
                  for i in range(b.n_psr)], axis=1) * np.sqrt(po["phi"])
    return np.einsum("rqj,rqj->rq", X[:, po["pairs"][:, 0]], X[:, po["pairs"][:, 1]])


def _map(pn, d):
    return d @ pn["V"][:pn["n_col"], :pn["kd"]].T / pn["dsqrt"]


def _check_max(res):
    """radio_snr_max / radio_argmax are the max and the first argmax of radio_snr."""
    import torch
    m = res["radio_snr"]
    assert torch.equal(res["radio_snr_max"], m.max(dim=1).values)
    first = torch.argmax((m == m.max(dim=1, keepdim=True).values).to(torch.int8), dim=1)
    assert torch.equal(res["radio_argmax"], first)
    assert int(res["radio_argmax"].max()) < m.shape[1]


def test_device_matches_plan_statics_ng15_full():
    psrs, noise = _ng15()
    b = _batch(psrs, noise)
    b.set_os_anisotropy(lmax=6, nside=8)
    pl = b.plan()
    po, pn = pl["os"], pl["os_aniso"]
    rows = b.generate(64, seed=SEED)
    got = b.optimal_statistic_of(rows, aniso_maps=True)
    ref = _map(pn, _pair_d(b, po, rows.cpu().numpy()))
    n_lm, n_z = pn["n_lm"], pn["n_z"]
    zr = ref[:, n_lm:n_lm + n_z]
    e_c = float(np.max(np.abs(got["clm"].cpu().numpy() - ref[:, :n_lm]) / np.sqrt(np.diag(pn["clm_cov"]))))
    e_z = float(np.max(np.abs(got["aniso_z"].cpu().numpy() - zr)))
    e_x = float(np.max(np.abs(got["aniso_chi2"].cpu().numpy() - np.sum(zr**2, axis=1)) /
                       np.maximum(np.sqrt(2.0 * n_z), np.sum(zr**2, axis=1))))
    e_r = float(np.max(np.abs(got["radio_snr"].cpu().numpy() - ref[:, n_lm + n_z:])))
    print(f"\n[os aniso] device vs numpy, 64 ng15-full rows, lmax 6 + nside 8 ({pn['n_col']} columns): |dc^|/sigma {e_c:.1e}, "
          f"|dz| {e_z:.1e}, chi2 rel {e_x:.1e}, |dS/N| {e_r:.1e}; statics {pn['setup_s']:.2f} s, cond(F) "
          f"{np.linalg.cond(pn['F'] / np.sqrt(np.outer(np.diag(pn['F']), np.diag(pn['F'])))):.1f}")
    assert e_c <= 1e-10 and e_z <= 1e-10 and e_x <= 1e-10 and e_r <= 1e-10
    _check_max(got)
    assert got["clm_lm"] == pn["clm_lm"] and np.array_equal(got["clm_cov"].cpu().numpy(), pn["clm_cov"])
    assert np.array_equal(got["radio_sigma"].cpu().numpy(), pn["radio_sigma"])
    assert np.array_equal(got["radio_sky"].cpu().numpy(), pn["sky"])
    # without aniso_maps the summaries are the same and no map is returned
    import torch
    lean = b.optimal_statistic_of(rows)
    assert "radio_snr" not in lean
    for k in ANISO_KEYS[:-1]:
        assert torch.equal(lean[k], got[k]), k
    # lmax 0: c^_00 = sqrt(4 pi) A2[hd]
    b.set_os_anisotropy(lmax=0)
    r0 = b.optimal_statistic_of(rows)
    e0 = float(np.max(np.abs(r0["clm"][:, 0].cpu().numpy() - np.sqrt(4 * np.pi) * r0["A2"][:, 0].cpu().numpy())) /
               (np.sqrt(4 * np.pi) * float(r0["A2_sigma"][0])))
    print(f"[os aniso] lmax 0: |c^_00 - sqrt(4 pi) A2[hd]| / sigma {e0:.1e}")
    assert e0 <= 1e-10 and r0["aniso_z"].shape == (64, 0) and float(r0["aniso_chi2"].abs().max()) == 0.0


def test_existing_outputs_unchanged_and_bit_identity():
    import torch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise)
    b.set_os_null("sky_scramble", n=100, seed=2)
    R = 1024
    base = b.optimal_statistic(R, seed=SEED, pairs=True, null_values=True)
    b.set_os_anisotropy(lmax=2, nside=4)
    a = b.optimal_statistic(R, seed=SEED, chunk=1024, pairs=True, null_values=True, aniso_maps=True)
    for k, v in base.items():
        if torch.is_tensor(v):
            assert torch.equal(a[k], v), k
    c = b.optimal_statistic(R, seed=SEED, chunk=256, aniso_maps=True)
    lo = b.optimal_statistic(512, seed=SEED, real0=0, aniso_maps=True)
    hi = b.optimal_statistic(512, seed=SEED, real0=512, aniso_maps=True)
    for k in ANISO_KEYS:
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    _check_max(a)
    b2 = _batch(psrs, noise, tm=False)
    b2.set_os_anisotropy(lmax=2, nside=4)
    e = b2.optimal_statistic(R, seed=SEED, aniso_maps=True)
    f = b2.optimal_statistic_of(b2.generate(R, seed=SEED), aniso_maps=True)
    for k in ANISO_KEYS:
        assert torch.equal(e[k], f[k]), k
    with pytest.raises(ValueError, match="radiometer"):
        b2.set_os_anisotropy(lmax=1)
        b2.optimal_statistic(4, aniso_maps=True)


def test_exact_noise_law_ng15_full():
    """No GWB, P = the generating model: cov(c^) = F^{-1}, z ~ N(0, I), E[chi2] = n_lm - 1, S/N_k ~ N(0, 1) with
    corr(S/N_k, S/N_k') = F_kk' / sqrt(F_kk F_k'k')."""
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False)
    b.set_os_anisotropy(lmax=6, nside=8)
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 3, aniso_maps=True)
    pn = b.plan()["os_aniso"]
    c, z, chi2, s = (res[k].cpu().numpy() for k in ("clm", "aniso_z", "aniso_chi2", "radio_snr"))
    sc = np.sqrt(np.diag(pn["clm_cov"]))
    cm, cv = np.abs(c.mean(axis=0)) / sc, c.var(axis=0, ddof=1) / sc**2
    cc = np.corrcoef(c.T)
    pc = pn["clm_cov"] / np.outer(sc, sc)
    n_z = pn["n_z"]
    t = b.plan()["os"]["t_ab"]
    Tr = pn["T_radio"]
    ks = [(0, 1), (0, 100), (300, 301), (5, 700), (400, 650)]
    pred = np.array([(Tr[i] * Tr[j]) @ t / np.sqrt(pn["radio_F"][i] * pn["radio_F"][j]) for i, j in ks])
    emp = np.array([np.corrcoef(s[:, i], s[:, j])[0, 1] for i, j in ks])
    print(f"\n[os aniso] noise law R={R}: c^ |mean|/sigma <= {cm.max():.4f}, var/F^-1 {cv.min():.3f}..{cv.max():.3f}, "
          f"max |corr - pred| {np.abs(cc - pc).max():.4f}; z |mean| <= {np.abs(z.mean(0)).max():.4f}, var "
          f"{z.var(0, ddof=1).min():.3f}..{z.var(0, ddof=1).max():.3f}; mean chi2 {chi2.mean():.3f} (n_z {n_z}); S/N "
          f"|mean| <= {np.abs(s.mean(0)).max():.4f}, var {s.var(0, ddof=1).min():.3f}..{s.var(0, ddof=1).max():.3f}; "
          f"pixel corr pred {np.round(pred, 3)} emp {np.round(emp, 3)}")
    assert np.all(cm < 4.5 / np.sqrt(R)) and np.all(np.abs(cv - 1) < 0.1)
    assert np.abs(cc - pc).max() < 5 / np.sqrt(R)
    assert np.all(np.abs(z.mean(0)) < 4.5 / np.sqrt(R)) and np.all(np.abs(z.var(0, ddof=1) - 1) < 0.1)
    assert abs(chi2.mean() - n_z) < 4 * np.sqrt(2.0 * n_z / R)
    assert np.all(np.abs(s.mean(0)) < 5 / np.sqrt(R)) and np.all(np.abs(s.var(0, ddof=1) - 1) < 0.12)
    assert np.all(np.abs(emp - pred) < 5 / np.sqrt(R))


def _clm_draw(B, scale, seed):
    """clm[0] = sqrt(4 pi), clm[1:] ~ scale N(0, 1), redrawn until sum c B is positive definite (bench config 4)."""
    rng = np.random.default_rng(seed)
    for _ in range(100):
        c = np.r_[np.sqrt(4 * np.pi), scale * rng.standard_normal(len(B) - 1)]
        if np.all(np.linalg.eigvalsh(sum(x * m for x, m in zip(c, B))) > 0):
            return c
    raise RuntimeError("no positive-definite ORF in 100 draws")


def test_injection_in_the_statistics_basis():
    """Rows + F_a c_a with c ~ N(0, A^2 Gamma (x) phi~), Gamma = sum c_lm B_lm (l <= lmax), drawn on the host in the
    statistic's own basis: E[d_q] = A^2 Gamma_q t_q, so E[c^] = A^2 c exactly and E[S/N_k] = A^2 T_k (Gamma t) / sqrt(F_kk)."""
    import torch
    from pta_replicator_b200 import orf
    psrs, noise = _ng15(npsr=12)
    b = _batch(psrs, noise, gwb=False, tm=False)
    lmax, K, log10_A = 2, 14, -14.0
    b.set_os_anisotropy(lmax=lmax, nside=4)
    pl = b.plan()
    po, pn = pl["os"], pl["os_aniso"]
    o = b._os
    locs = orf.psrlocs_from_pulsars(b.psrs)
    B = orf.correlated_basis(np.stack([locs[:, 0], np.pi / 2 - locs[:, 1]], axis=1), lmax)
    c = _clm_draw(B, 0.6, 3)
    Gam = sum(x * m for x, m in zip(c, B))
    mu, E = np.linalg.eigh(Gam)
    Bm = E * np.sqrt(mu)
    sp = np.sqrt(OO.phi_tilde(K, o["gamma"], o["Tspan"]))
    Fg = [OO.gw_basis(b.t_tdb[i], K, o["Tspan"]) for i in range(b.n_psr)]
    R, chunk = 4096, 512
    rng = np.random.default_rng(17)
    outs = []
    for r0 in range(0, R, chunk):
        rows = b.generate(chunk, seed=SEED + 9, real0=r0).cpu().numpy()
        cc = 10.0 ** log10_A * np.einsum("ab,rbi->rai", Bm, rng.standard_normal((chunk, b.n_psr, 2 * K))) * sp
        for i in range(b.n_psr):
            s, n = b.toa_off[i], b.ntoa[i]
            rows[:, s:s + n] += cc[:, i] @ Fg[i].T
        res = b.optimal_statistic_of(torch.from_numpy(rows).to(b.device), aniso_maps=True)
        outs.append(np.concatenate([res["clm"].cpu().numpy(), res["radio_snr"].cpu().numpy()], axis=1))
    got = np.concatenate(outs)
    A2 = 10.0 ** (2 * log10_A)
    ed = A2 * Gam[po["pairs"][:, 0], po["pairs"][:, 1]] * po["t_ab"]
    exp = np.r_[A2 * c, (_map(pn, ed[None])[0])[pn["n_lm"] + pn["n_z"]:]]
    zs = (got.mean(axis=0) - exp) / (got.std(axis=0, ddof=1) / np.sqrt(R))
    print(f"\n[os aniso] own-basis injection R={R}: E[c^]/A^2 = {np.round(c, 3)}; mean c^/A^2 "
          f"{np.round(got[:, :len(c)].mean(0) / A2, 3)}; max |(mean - E) / se| c^ {np.abs(zs[:len(c)]).max():.2f}, "
          f"S/N {np.abs(zs[len(c):]).max():.2f} (E[S/N] up to {exp[len(c):].max():.2f})")
    assert np.all(np.abs(zs[:len(c)]) < 4) and np.all(np.abs(zs[len(c):]) < 4.5)


def test_set_gwb_anisotropic_injection_matches_oracle_ng15_epoch():
    """``set_gwb(lmax=6, clm=...)`` (the config-4 draw) at ng15-epoch: mean c^ and mean radiometer S/N against the dense
    oracle's exact expectation (E[d_q] from the injection covariance, then its least-squares fit and radiometer)."""
    from pta_replicator_b200 import orf
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=False, tm=True)
    locs = orf.psrlocs_from_pulsars(b.psrs)
    B = orf.correlated_basis(np.stack([locs[:, 0], np.pi / 2 - locs[:, 1]], axis=1), 6)
    clm = _clm_draw(B, 0.05, 20250922)
    b.set_gwb(-14.0, 13.0 / 3.0, lmax=6, clm=list(clm))
    b.set_os_anisotropy(lmax=6, nside=8)
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 5, aniso_maps=True)
    models = []
    for i, p in enumerate(b.psrs):
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        models.append(TO.timing_design_matrix(t, 2, [f.get("f") for f in p.toas.table["flags"]])[b.order[i]])
    S = OO.statics(b, models=models, templates=("hd",))
    ed = AO.expected_pair_means(b, S)
    pa, pb = S["pairs"]
    t = S["t"][pa, pb]
    ec, _ = AO.sph_fit(ed[None], t, AO.sph_templates(b, 6, S["pairs"]))
    es, _ = AO.radiometer(ed[None], t, AO.radio_templates(b, res["radio_sky"].cpu().numpy(), S["pairs"]))
    exp = np.r_[ec[0], es[0]]
    got = np.concatenate([res["clm"].cpu().numpy(), res["radio_snr"].cpu().numpy()], axis=1)
    zs = (got.mean(axis=0) - exp) / (got.std(axis=0, ddof=1) / np.sqrt(R))
    print(f"\n[os aniso] set_gwb lmax 6 at ng15-epoch, R={R}: E[c^_00] {exp[0]:.3e}, max E[S/N] {es.max():.2f}; "
          f"max |(mean - E) / se| c^ {np.abs(zs[:49]).max():.2f}, S/N {np.abs(zs[49:]).max():.2f}")
    assert np.all(np.abs(zs[:49]) < 4) and np.all(np.abs(zs[49:]) < 4.5)


# ------------------------------------------------------------------ edge sweep
EDGE_CASES = [  # (P, lmax, S (None: no radiometer; 'nside n'), R)
    (2, 0, 1, 1), (3, 0, 12, 1025), (3, None, 12288, 65), (67, 6, 768, 65), (67, 7, 3072, 1),
    (24, 1, 12288, 65), (256, 7, None, 1), (256, None, 12, 65), (67, 0, None, 1025)]
REPORT = RR.Report()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[edges] anisotropy:\n  " + "\n  ".join(REPORT.lines()))


@pytest.mark.parametrize("P,lmax,S,R", EDGE_CASES)
def test_os_aniso_edges(P, lmax, S, R):
    """Every output within its rigorous bound from the extended-precision reference on the device's own statics
    (V, dsqrt as uploaded): the map columns as ptar_os_null's sky-scramble GEMM, chi2 = sum z^2 with its propagated
    bound, max / argmax where the top two are farther apart than their bounds, and no argmax >= S."""
    import torch
    from pta_replicator_b200.engine import healpix_ring_centres
    from tests.test_gpu_reduction_edges import _os_statics, _rows, _t
    rng = np.random.default_rng(P)
    ntoas = (5, 65) if P == 2 else RR.null_ntoas(P) if P <= 24 else tuple(int(n) for n in rng.integers(8, 41, P))
    b = RR.edge_batch(ntoas, seed=300 + P, tm_min=24)
    b.set_optimal_statistic(components=5, orfs=("hd",))
    sky = None
    if S is not None:
        nside = {12: 1, 768: 8, 3072: 16, 12288: 32}.get(S)
        sky = healpix_ring_centres(nside) if nside else np.array([[1.1, 0.4]])
    b.set_os_anisotropy(lmax=lmax, sky=sky)
    rows = _rows(b, R, seed=P + R)
    res = b.optimal_statistic_of(_t(b, rows), aniso_maps=S is not None)
    st = b.compile()["os"]["aniso"]
    am = st["model"]
    N = dict(method="sky_scramble", V=st["dev"]["V"].cpu().numpy().reshape(am.n_colp, am.kdp), kd=am.kd, n_col=am.n_col,
             dsqrt=st["dev"]["dsqrt"].cpu().numpy())
    Sd = _os_statics(b)
    ref = RR.os_null(Sd, N, RR.optimal_statistic(Sd, rows))["snr"]
    n_lm, n_z, tag = am.n_lm, am.n_z, f"P={P} lmax={lmax} S={S} R={R}"
    sl = lambda a, b_: {k: v[:, a:b_] for k, v in ref.items()}          # noqa: E731
    if n_lm:
        RR.check(res["clm"].cpu().numpy(), sl(0, n_lm), f"{tag} c^", REPORT, "aniso_clm")
        zr = sl(n_lm, n_lm + n_z)
        if n_z:
            RR.check(res["aniso_z"].cpu().numpy(), zr, f"{tag} z", REPORT, "aniso_z")
        zv = zr["hi"].astype(np.longdouble) + zr["lo"]
        ch = np.sum(zv * zv, axis=1)
        cb = np.sum(2 * np.abs(zr["hi"]) * zr["bound"] + zr["bound"] ** 2, axis=1) + RR.gamma(n_z + 8) * np.sum(zr["hi"] ** 2, axis=1)
        chh = ch.astype(np.float64)
        RR.check(res["aniso_chi2"].cpu().numpy(), dict(hi=chh, lo=(ch - chh).astype(np.float64), bound=cb,
                                                       terms=np.sum(zr["hi"] ** 2, axis=1)),
                 f"{tag} chi2", REPORT, "aniso_chi2")
    if S is not None:
        rr = sl(n_lm + n_z, n_lm + n_z + S)
        RR.check(res["radio_snr"].cpu().numpy(), rr, f"{tag} radiometer S/N", REPORT, "aniso_radio")
        _check_max(res)
        am_ = res["radio_argmax"].cpu().numpy()
        assert np.all((am_ >= 0) & (am_ < S))
        if S > 1:
            srt = np.sort(rr["hi"], axis=1)
            top = np.argmax(rr["hi"], axis=1)
            clear = (srt[:, -1] - srt[:, -2]) > 2 * rr["bound"].max(axis=1)
            assert np.array_equal(am_[clear], top[clear])
    # staged launches equal the fused ones
    again = b.optimal_statistic_of(_t(b, rows), aniso_maps=S is not None, timers={})
    for k in ANISO_KEYS:
        if k in res:
            assert torch.equal(res[k], again[k]), k
