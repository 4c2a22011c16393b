"""GPU tests of the per-frequency optimal statistic (``PulsarBatch.set_os_per_frequency`` -> ``ptar_os_pf``): the device
against the plan's statics applied in numpy, existing outputs unchanged by the registration, bit-identity across
chunking, real0 splits and paths, the numerator identity with the broadband statistic, the exact noise law, the
recovered spectrum of a turnover injection against the dense oracle's exact expectation, and edge shapes through the
C ABI against an extended-precision restatement on the same projections."""
import ctypes as C

import numpy as np
import pytest

from tests import os_oracle as OO
from tests import pfos_oracle as PO
from tests import reduction_reference as RR
from tests import timing_oracle as TO
from tests.test_gpu_optimal_statistic import SEED, _batch, _ng15

pytestmark = pytest.mark.gpu

PF_KEYS = ("pf_phi", "pf_snr", "pf_phi_mc", "pf_rho")
PF_STATIC = ("pf_freqs", "pf_phi_tilde", "pf_sigma", "pf_phi_sigma", "pf_cov_mc")


def _numpy_pf(b, po, pp, rows):
    """The plan's statics applied with numpy to host rows [R, ld]."""
    nc = po["nc"]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :nc]
                  for i in range(b.n_psr)], axis=1)
    return _pf_of_X(po, pp, X)


def _pf_of_X(po, pp, X):
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    R, K = X.shape[0], pp["K"]
    d = (X[:, pa, :2 * K] * X[:, pb, :2 * K]).reshape(R, len(pa), K, 2).sum(axis=3).transpose(0, 2, 1)
    bo = np.einsum("oq,rkq->rok", po["orf"], d)
    return dict(pf_rho=d / pp["t"], pf_phi=bo / pp["dnorm"], pf_snr=bo / pp["dsqrt"],
                pf_phi_mc=np.einsum("kop,rpk->rok", pp["finv"], bo), b=bo)


def _np(t):
    return t.cpu().numpy()


def test_device_matches_numpy_and_numerator_identity_ng15_full():
    psrs, noise = _ng15()
    b = _batch(psrs, noise)
    b.set_os_per_frequency()
    pl = b.plan()
    po, pp = pl["os"], pl["os_pf"]
    rows = b.generate(64, seed=SEED)                       # post-fit rows (spin + JUMPs)
    got = b.optimal_statistic_of(rows, pairs=True)
    ref = _numpy_pf(b, po, pp, rows.cpu().numpy())
    sig_mc = np.sqrt(np.stack([np.diag(f) for f in pp["finv"]], axis=1))
    e = dict(rho=float(np.max(np.abs(_np(got["pf_rho"]) - ref["pf_rho"]) / pp["sigma"])),
             phi=float(np.max(np.abs(_np(got["pf_phi"]) - ref["pf_phi"]) / pp["phi_sigma"])),
             snr=float(np.max(np.abs(_np(got["pf_snr"]) - ref["pf_snr"]))),
             phi_mc=float(np.max(np.abs(_np(got["pf_phi_mc"]) - ref["pf_phi_mc"]) / sig_mc)))
    print(f"\n[os pf] device vs numpy, 64 ng15-full rows, K={pp['K']}, {len(po['t_ab'])} pairs: " +
          ", ".join(f"|d{k}|/sigma {v:.1e}" for k, v in e.items()) + f"; statics {pp['setup_s']:.2f} s")
    assert max(e.values()) <= 1e-10
    assert got["pf_rho"].shape == (64, pp["K"], len(po["t_ab"])) and got["pf_phi"].shape == (64, 3, pp["K"])
    for k, key in zip(PF_STATIC, ("freqs", "phi_tilde", "sigma", "phi_sigma", "finv")):
        assert np.array_equal(_np(got[k]), pp[key]), k
    assert got["pf_setup_s"] == b.os_pf_setup_s           # the plan() of compile()
    # sum_k phi~_k b_ok = b_o = A2_o D_o, every quantity rebuilt from the returned outputs
    bk = _np(got["pf_phi"]) / _np(got["pf_phi_sigma"]) ** 2
    ph = _np(got["pf_phi_tilde"])
    num = np.einsum("k,rok->ro", ph, bk)
    mag = np.einsum("k,rok->ro", ph, np.abs(bk))
    bo = _np(got["A2"]) / _np(got["A2_sigma"]) ** 2
    e_id = float(np.max(np.abs(num - bo) / mag))
    print(f"[os pf] numerator identity: max |sum_k phi~_k b_ok - A2_o D_o| / sum_k |phi~_k b_ok| = {e_id:.1e}")
    assert e_id <= 1e-12


def test_existing_outputs_unchanged_and_bit_identity():
    import torch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise)
    b.set_os_null("sky_scramble", n=100, seed=2)
    b.set_os_anisotropy(lmax=2, nside=4)
    R = 1024
    base = b.optimal_statistic(R, seed=SEED, pairs=True, null_values=True, aniso_maps=True)
    assert not any(k.startswith("pf_") for k in base)
    b.set_os_per_frequency()
    a = b.optimal_statistic(R, seed=SEED, chunk=1024, pairs=True, null_values=True, aniso_maps=True)
    for k, v in base.items():
        if torch.is_tensor(v):
            assert torch.equal(a[k], v), k
    c = b.optimal_statistic(R, seed=SEED, chunk=256, pairs=True)
    lo = b.optimal_statistic(512, seed=SEED, real0=0, pairs=True)
    hi = b.optimal_statistic(512, seed=SEED, real0=512, pairs=True)
    for k in PF_KEYS:
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    lean = b.optimal_statistic(R, seed=SEED)
    assert "pf_rho" not in lean
    for k in PF_KEYS[:-1]:
        assert torch.equal(lean[k], a[k]), k
    timed = {}
    b.optimal_statistic(256, seed=SEED, timers=timed)
    assert "os_pf" in {name for name, _, _ in timed["events"]}
    b2 = _batch(psrs, noise, tm=False)
    b2.set_os_per_frequency()
    e = b2.optimal_statistic(R, seed=SEED, pairs=True)
    f = b2.optimal_statistic_of(b2.generate(R, seed=SEED), pairs=True)
    for k in PF_KEYS:
        assert torch.equal(e[k], f[k]), k


def _snr_kurtosis(po, pp):
    """Excess kurtosis [n_orf, K] of S/N_ok under the noise model.  S/N_ok = x^T A x with x = (X_a,k)_a ~ N(0, Sigma),
    Sigma = blockdiag(Z_a[k]), A_ab = Gamma^o_ab I_2 / (2 sqrt(D_ok)) (a != b): its cumulants are 2^(r-1) (r-1)!
    tr((A Sigma)^r), so var = 2 tr((A Sigma)^2) = 1 and excess kurtosis = 48 tr((A Sigma)^4)."""
    P, K = po["Z"].shape[0], pp["K"]
    Z = po["Z"].reshape(P, K, 2, K, 2)[:, np.arange(K), :, np.arange(K), :]
    Z = 0.5 * (Z + Z.transpose(0, 1, 3, 2))
    out = np.empty(pp["dnorm"].shape)
    for o in range(out.shape[0]):
        G = np.zeros((P, P))
        G[po["pairs"][:, 0], po["pairs"][:, 1]] = po["orf"][o]
        G = G + G.T
        for k in range(K):
            M = np.einsum("ab,bij->aibj", G, Z[k]).reshape(2 * P, 2 * P) / (2 * np.sqrt(pp["dnorm"][o, k]))
            M2 = M @ M
            assert abs(2 * np.trace(M2) - 1) < 1e-9
            out[o, k] = 48 * np.trace(M2 @ M2)
    return out


def test_noise_law_ng15_full():
    """No GWB, P = the generating model: S/N_ok has mean 0 and unit variance at every (o, k) (pairs sharing a pulsar
    are uncorrelated), rho_qk / sigma_qk unit variance.  S/N_ok is a quadratic form of Gaussians, not a Gaussian: its
    excess kurtosis kappa (1.2 .. 10 here, largest for the monopole at f_1) sets the standard error of a sample
    variance, sqrt((2 + kappa) / R), so the variance is checked at 4.5 of those standard errors."""
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False)
    b.set_os_per_frequency()
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 3, pairs=True)
    pl = b.plan()
    kap = _snr_kurtosis(pl["os"], pl["os_pf"])
    s = _np(res["pf_snr"])
    mean, var = s.mean(axis=0), s.var(axis=0, ddof=1)
    se_var = np.sqrt((2 + kap) / R)
    z = res["pf_rho"] / res["pf_sigma"]
    pooled = float(z.var())
    del z
    print(f"\n[os pf] noise law R={R}: S/N |mean| <= {np.abs(mean).max():.4f} (bound {4 / np.sqrt(R):.4f}), var "
          f"{var.min():.3f}..{var.max():.3f}, max |var - 1| / se {np.max(np.abs(var - 1) / se_var):.2f} (excess kurtosis "
          f"{kap.min():.2f}..{kap.max():.2f}); pooled rho/sigma var {pooled:.4f}")
    assert np.all(np.abs(mean) < 4 / np.sqrt(R))
    assert np.all(np.abs(var - 1) < 4.5 * se_var)
    assert abs(pooled - 1) < 5 * np.sqrt(2.0 / R)


def test_turnover_spectrum_recovered_ng15_epoch():
    """A GWB with a low-frequency turnover (hc / (1 + (f / f0)^(-5/3)), f0 = 4 nHz), which the broadband statistic's
    power-law shape cannot follow: the mean of pf_phi for HD at every f_k within 4 standard errors of the dense
    oracle's exact E[phi_k] from the injection covariance."""
    from pta_replicator_b200 import constants as const
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=False, tm=True)
    log10_A, f0 = -14.6733, 4e-9
    b.set_gwb(log10_A, 13.0 / 3.0, turnover=True, f0=f0)
    b.set_os_per_frequency()
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 5)
    phi = _np(res["pf_phi"])[:, 0]
    models = []
    for i, p in enumerate(b.psrs):
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        models.append(TO.timing_design_matrix(t, 2, [f.get("f") for f in p.toas.table["flags"]])[b.order[i]])
    S = OO.statics(b, models=models)
    T = PO.pf_statics(b, S)
    e = PO.expected_pf_phi(b, S, T)[0]
    m, se = phi.mean(axis=0), phi.std(axis=0, ddof=1) / np.sqrt(R)
    f = _np(res["pf_freqs"])
    alpha = -2.0 / 3.0
    hc = 10**log10_A * (f / const.GWB_F1YR) ** alpha / (1 + (f / f0) ** (alpha - 1))
    inj = hc**2 / (12 * np.pi**2 * f**3 * b._os["Tspan"])
    pl = 10 ** (2 * log10_A) * _np(res["pf_phi_tilde"])
    print(f"\n[os pf] turnover injection R={R}, f0 = {f0:.0e} Hz:\n  k  f [nHz]  mean/injected  E/injected  "
          f"injected/power-law  (mean - E)/se")
    for k in range(len(f)):
        print(f"  {k + 1:2d}  {f[k] * 1e9:6.2f}  {m[k] / inj[k]:12.3f}  {e[k] / inj[k]:10.3f}  {inj[k] / pl[k]:17.3f}  "
              f"{(m[k] - e[k]) / se[k]:+6.2f}")
    assert np.all(np.abs(m - e) < 4 * se)
    assert inj[0] / pl[0] < 0.1                           # the turnover is strong where the test looks


# ------------------------------------------------------------------ edge shapes through the C ABI
EDGE_CASES = [  # (P, K, n_orf, R)
    (2, 1, 1, 3), (2, 16, 1, 65), (3, 1, 1, 1), (24, 16, 4, 65), (24, 5, 1, 130), (67, 14, 4, 33), (140, 16, 1, 9),
    (140, 3, 4, 64), (256, 16, 4, 5)]


def _pf_longdouble(po, pp, X):
    """Extended-precision outputs of the device's own X and statics, and the componentwise bound of a fp64 evaluation
    (gamma_n u = n u / (1 - n u) per sum of n products)."""
    L = np.longdouble
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    R, K, Q = X.shape[0], pp["K"], len(pa)
    Xl = X[:, :, :2 * K].astype(L)
    prod = (Xl[:, pa] * Xl[:, pb]).reshape(R, Q, K, 2)
    d = prod.sum(axis=3).transpose(0, 2, 1)
    ad = np.abs(prod).sum(axis=3).transpose(0, 2, 1)
    W = po["orf"].astype(L)
    bo = np.einsum("oq,rkq->rok", W, d)
    M = np.einsum("oq,rkq->rok", np.abs(W), ad)
    u = 2.0**-53
    g = lambda n: n * u / (1 - n * u)                                   # noqa: E731
    bb = g(Q + 2) * M                                                   # |b_fp64 - b|
    Fi = pp["finv"].astype(L)
    return dict(pf_rho=(d / pp["t"], g(3) * ad / pp["t"] + u * np.abs(d / pp["t"])),
                pf_phi=(bo / pp["dnorm"], bb / pp["dnorm"] + u * np.abs(bo / pp["dnorm"])),
                pf_snr=(bo / pp["dsqrt"], bb / pp["dsqrt"] + u * np.abs(bo / pp["dsqrt"])),
                pf_phi_mc=(np.einsum("kop,rpk->rok", Fi, bo),
                           np.einsum("kop,rpk->rok", np.abs(Fi), bb) * (1 + g(5)) +
                           g(5) * np.einsum("kop,rpk->rok", np.abs(Fi), np.abs(bo))))


@pytest.mark.parametrize("P,K,n_orf,R", EDGE_CASES)
def test_os_pf_edges(P, K, n_orf, R):
    """Every output within its rigorous bound of the extended-precision evaluation on the device's own projections X
    (``ptar_os_project``'s, read back) and uploaded statics; ``ptar_os_pf`` called directly equals
    ``optimal_statistic_of`` bit for bit; a NaN in one row leaves every other realization bit-identical."""
    import torch
    from pta_replicator_b200 import _cabi
    from tests.test_gpu_reduction_edges import _rows, _t
    rng = np.random.default_rng(P + K)
    ntoas = (5, 65) if P == 2 else RR.null_ntoas(P) if P <= 24 else tuple(int(n) for n in rng.integers(8, 41, P))
    b = RR.edge_batch(ntoas, seed=400 + P, tm_min=24)
    b.set_optimal_statistic(components=K, orfs=RR.templates(P, "hd" if n_orf == 1 else "all4"))
    b.set_os_per_frequency()
    rows = _rows(b, R, seed=P + R)
    res = b.optimal_statistic_of(_t(b, rows), pairs=True)
    pl = b.plan()
    po, pp = pl["os"], pl["os_pf"]
    st = b.compile()["os"]
    # X of the same rows on the device, then the entry point on it
    X = b._os_project(st, _t(b, rows), R, None)[:R * P * po["ncp"]].clone()
    out = {k: torch.empty_like(res[k]) for k in PF_KEYS}
    L = _cabi.lib()
    _cabi.check(L.ptar_os_pf(X.data_ptr(), R, C.byref(st["model"]), C.byref(st["pf"]["model"]), out["pf_rho"].data_ptr(),
                             out["pf_phi"].data_ptr(), out["pf_snr"].data_ptr(), out["pf_phi_mc"].data_ptr(),
                             _cabi.current_stream()), "ptar_os_pf")
    torch.cuda.synchronize()
    for k in PF_KEYS:
        assert torch.equal(out[k], res[k]), k
    ref = _pf_longdouble(po, pp, X.cpu().numpy().reshape(R, P, po["ncp"]))
    worst = {}
    for k, (v, bound) in ref.items():
        err = np.abs(_np(res[k]).astype(np.longdouble) - v)
        assert np.all(err <= 2 * bound), (k, float(np.max(err - 2 * bound)))
        worst[k] = float(np.max(err / np.maximum(bound, np.finfo(float).tiny)))
    print(f"\n[os pf edges] P={P} K={K} n_orf={n_orf} R={R}: max err / bound " +
          ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    # a NaN in one TOA of one realization: that realization's statistics are not finite, the others are unchanged
    r_bad = R // 2
    poisoned = rows.copy()
    poisoned[r_bad, b.toa_off[P - 1]] = np.nan
    pz = b.optimal_statistic_of(_t(b, poisoned), pairs=True)
    keep = [r for r in range(R) if r != r_bad]
    for k in PF_KEYS:
        assert torch.equal(pz[k][keep], res[k][keep]), k
    assert not torch.isfinite(pz["pf_phi"][r_bad]).any() and not torch.isfinite(pz["pf_snr"][r_bad]).any()
    assert not torch.isfinite(pz["pf_phi_mc"][r_bad]).any()
    last = torch.from_numpy(po["pairs"][:, 1] == P - 1).to(b.device)
    assert not torch.isfinite(pz["pf_rho"][r_bad][:, last]).any()
    assert torch.equal(pz["pf_rho"][r_bad][:, ~last], res["pf_rho"][r_bad][:, ~last])
