"""GPU tests of the Fp-statistic (``PulsarBatch.fp_statistic`` / ``fp_statistic_of`` -> ``ptar_fp_project`` +
``ptar_fp_reduce``): the device against the plan's statics in numpy on the same rows, pre-fit against post-fit rows,
bit-identity across chunking, real0 splits and paths, the exact null law (including the predicted correlation of
neighbouring frequencies) and an injected continuous wave against the dense oracle's noncentrality."""
import numpy as np
import pytest

from tests import fp_oracle as FO
from tests import reduction_reference as RR
from tests import timing_oracle as TO

pytestmark = pytest.mark.gpu

SEED = 20251015
NF = 100


def _ng15(kind="full", npsr=None):
    from pta_replicator_b200 import synthetic
    return synthetic.make_ng15_like(kind, npsr=npsr)


def _batch(psrs, noise, gwb=True, tm=True, **fp):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise, gwb=gwb)
    if tm:
        for i in range(b.n_psr):
            b.set_timing_model(i, poly=2, jumps="f")
    b.set_fp_statistic(**fp)
    return b


def _models(b):
    out = []
    for i, p in enumerate(b.psrs):                          # the oracle's own design matrices, engine order
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        out.append(TO.timing_design_matrix(t, 2, [f.get("f") for f in p.toas.table["flags"]])[b.order[i]])
    return out


def _statics(b):
    """The plan's Fp statics as the device holds them (one host derivation per batch: compile() runs plan())."""
    st = b.compile()["fp"]
    return dict(Ct=st["Ct"].cpu().numpy(), n_freq=st["n_freq"], freqs=st["out"]["freqs"].cpu().numpy(),
                M=st["out"]["M"].cpu().numpy(), setup_s=st["setup_s"])


@pytest.fixture(scope="module")
def full_gwb():
    psrs, noise = _ng15()
    b = _batch(psrs, noise, n_freqs=NF)
    return b, _statics(b)


def test_device_matches_numpy_and_fap_matches_q_ng15_full(full_gwb):
    """Fp and X^ against numpy on the same rows; fap within 1e-12 relative of Q(P, Fp) in extended precision."""
    import torch
    from pta_replicator_b200.engine import fp_whitened_basis
    b, pf = full_gwb
    rows = b.generate(64, seed=SEED)                        # post-fit rows (spin + JUMPs)
    got = b.fp_statistic_of(rows, pulsars=True)
    h = rows.cpu().numpy()
    amps = np.stack([h[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ fp_whitened_basis(pf, b.toa_off[i], b.ntoa[i])
                     for i in range(b.n_psr)], axis=1).reshape(64, b.n_psr, NF, 2)
    Fp = 0.5 * np.sum(amps**2, axis=(1, 3))
    d_amps = float(np.max(np.abs(got["amps"].cpu().numpy() - amps)))
    d_fp = float(np.max(np.abs(got["Fp"].cpu().numpy() - Fp)))
    print(f"\n[fp] device vs numpy, 64 realizations ng15-full Nf={NF}: |dFp| {d_fp:.1e} (bound {1e-10 * np.sqrt(b.n_psr):.1e}), "
          f"|damps| {d_amps:.1e}; host statics {pf['setup_s']:.1f} s; C~ {pf['Ct'].nbytes / 1e9:.2f} GB")
    assert d_fp <= 1e-10 * np.sqrt(b.n_psr) and d_amps <= 1e-10
    F = got["Fp"]
    assert torch.equal(got["Fp_max"], F.max(dim=1).values)
    assert np.array_equal(got["Fp_argmax"].cpu().numpy(), np.argmax(F.cpu().numpy(), axis=1))
    q = RR.q_int(b.n_psr, F.cpu().numpy().ravel(), np.longdouble).astype(float).reshape(F.shape)
    fap = got["fap"].cpu().numpy()
    keep = q >= 1e-300                                      # below, Q underflows (GWB rows reach Fp ~ 1e3)
    rel = float(np.max(np.abs(fap[keep] - q[keep]) / q[keep]))
    print(f"[fp] fap vs Q(P, Fp) in extended precision: worst relative error {rel:.1e}")
    assert rel <= 1e-12 and np.all(fap[~keep] <= 1e-290)
    assert np.array_equal(got["freqs"].cpu().numpy(), np.arange(1, NF + 1) / b._fp["Tspan"])
    assert got["M"].shape == (b.n_psr, NF, 2, 2)
    assert got["Fp_argmax"].dtype == torch.int64 and got["amps"].shape == (64, b.n_psr, NF, 2)


def test_prefit_statistic_equals_postfit_rows(full_gwb):
    """fp_statistic skips the timing fit: P^{-1} annihilates the timing columns."""
    b, _ = full_gwb
    R = 256
    a = b.fp_statistic(R, seed=SEED, pulsars=True)
    c = b.fp_statistic_of(b.generate(R, seed=SEED), pulsars=True)
    d_amps = float((a["amps"] - c["amps"]).abs().max())
    d_fp = float((a["Fp"] - c["Fp"]).abs().max())
    print(f"\n[fp] pre-fit vs post-fit rows: |damps| {d_amps:.1e} (sigma units), |dFp| {d_fp:.1e}; "
          f"max |amps| {float(a['amps'].abs().max()):.1f}")
    assert d_amps <= 1e-9


def test_unregistered_batch_raises():
    psrs, noise = _ng15("epoch", npsr=4)
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise, gwb=False)
    with pytest.raises(ValueError, match="set_fp_statistic"):
        b.fp_statistic(8)
    with pytest.raises(ValueError, match="set_fp_statistic"):
        b.fp_statistic_of(b.generate(8))


def test_bit_identity_across_chunks_real0_and_paths():
    import torch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise, n_freqs=NF)
    R = 1024
    a = b.fp_statistic(R, seed=SEED, chunk=1024, pulsars=True)
    c = b.fp_statistic(R, seed=SEED, chunk=256, pulsars=True)
    lo = b.fp_statistic(512, seed=SEED, real0=0, pulsars=True)
    hi = b.fp_statistic(512, seed=SEED, real0=512, pulsars=True)
    for k in ("Fp", "Fp_max", "Fp_argmax", "fap", "amps"):
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    # without a timing model the generated rows are the rows the statistic reduces
    b2 = _batch(psrs, noise, tm=False, n_freqs=NF)
    e = b2.fp_statistic(R, seed=SEED, pulsars=True)
    f = b2.fp_statistic_of(b2.generate(R, seed=SEED), pulsars=True)
    for k in ("Fp", "Fp_max", "Fp_argmax", "fap", "amps"):
        assert torch.equal(e[k], f[k]), k


def test_null_law_ng15_full():
    """White + ECORR + RN with timing models, no GWB, P = the generating model: X^ ~ N(0, I), 2 Fp(f) ~ chi^2_2P, and
    neighbouring frequencies correlate as sum_a 2 |B_a|_F^2 / 4P, B_a = L_f^-1 F_f^T P_a^-1 F_f' L_f'^-T (exact in law)."""
    from pta_replicator_b200.engine import _sincos_basis, fp_whitened_basis
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False, n_freqs=NF)
    pf = _statics(b)
    P, R = b.n_psr, 4096
    res = b.fp_statistic(R, seed=SEED + 3, pulsars=True)
    x = 2.0 * res["Fp"].cpu().numpy()
    amps = res["amps"].cpu().numpy()
    mean, var = x.mean(axis=0), x.var(axis=0, ddof=1)
    am, av = float(amps.mean()), float(amps.var())
    corr = np.array([np.corrcoef(x[:, f], x[:, f + 1])[0, 1] for f in range(NF - 1)])
    pred = np.zeros(NF - 1)
    for i in range(P):
        F = _sincos_basis(b.t_tdb[i], pf["freqs"])
        Ct = fp_whitened_basis(pf, b.toa_off[i], b.ntoa[i])
        for f in range(NF - 1):
            L = np.linalg.cholesky(pf["M"][i, f])
            B = np.linalg.solve(L, F[:, 2 * f:2 * f + 2].T @ Ct[:, 2 * f + 2:2 * f + 4])
            pred[f] += 2.0 * np.sum(B * B) / (4.0 * P)
    zm = (mean - 2 * P) / np.sqrt(4 * P / R)
    print(f"\n[fp] null law R={R}, P={P}: mean 2Fp z in [{zm.min():.2f}, {zm.max():.2f}], var/4P in "
          f"[{(var / (4 * P)).min():.3f}, {(var / (4 * P)).max():.3f}]; amps mean {am:.4f} var {av:.4f}; neighbour corr "
          f"predicted {pred.min():.3f}..{pred.max():.3f}, max |measured - predicted| {np.max(np.abs(corr - pred)):.3f}")
    assert np.all(np.abs(zm) < 5)
    assert np.all(np.abs(var / (4 * P) - 1) < 0.1)
    assert abs(am) < 0.01 and abs(av - 1) < 0.05
    assert np.all(np.abs(corr - pred) < 5 / np.sqrt(R))
    assert np.all(res["fap"].cpu().numpy() >= 0) and np.all(res["fap"].cpu().numpy() <= 1)


def test_injected_cw_matches_oracle_noncentrality_ng15_epoch():
    """ng15-epoch (the dense oracle fits): a row holding only one add_cgw source gives 2 Fp = lambda_f of the oracle;
    with noise plus the same source, mean 2 Fp(f) = 2P + lambda_f within 4 standard errors at every f."""
    import torch
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=False, n_freqs=NF)
    P = b.n_psr
    src = dict(gwtheta=1.1, gwphi=2.3, mc=10**9.2, fgw=6.5 / b._fp["Tspan"], phase0=0.7, psi=0.4, inc=1.0)
    d1 = b.cgw_delays(dist=1.0, **src)                     # residuals scale as 1 / dist
    S = FO.statics(b, b._fp["freqs"], models=_models(b))
    row1 = np.zeros(b.ld)
    for i in range(P):
        row1[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = d1[i]
    lam1 = FO.noncentrality(b, S, row1)
    dist = float(np.sqrt(lam1.max() / 150.0))              # peak lambda_f = 150
    d = b.cgw_delays(dist=dist, **src)
    row = np.zeros(b.ld)
    for i in range(P):
        row[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = d[i]
    lam = FO.noncentrality(b, S, row)
    got = 2.0 * b.fp_statistic_of(torch.from_numpy(row[None, :]).to(b.device))["Fp"].cpu().numpy()[0]
    rel = float(np.max(np.abs(got - lam) / lam))
    b.add_cgw(dist=dist, **src)
    R = 4096
    x = 2.0 * b.fp_statistic(R, seed=SEED + 5)["Fp"].cpu().numpy()
    se = np.sqrt(2.0 * (2 * P + 2 * lam) / R)
    z = (x.mean(axis=0) - (2 * P + lam)) / se
    k = int(np.argmax(lam))
    print(f"\n[fp] CW on ng15-epoch: max |2Fp - lambda| / lambda {rel:.1e}; peak lambda {lam[k]:.1f} at f index {k}; "
          f"z of mean 2Fp in [{z.min():.2f}, {z.max():.2f}], at the peak {z[k]:.2f}")
    assert rel <= 1e-10
    assert np.all(np.abs(z) < 4)
