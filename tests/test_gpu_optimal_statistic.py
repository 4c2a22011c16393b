"""GPU tests of the optimal statistic (``PulsarBatch.optimal_statistic`` / ``optimal_statistic_of`` ->
``ptar_os_project`` + ``ptar_os_pairs``): the device against numpy on the same rows, pre-fit against post-fit rows,
bit-identity across chunking, real0 splits and paths, the null law and the injected-signal mean against the dense
oracle's exact expectation."""
import numpy as np
import pytest

from tests import os_oracle as OO
from tests import timing_oracle as TO

pytestmark = pytest.mark.gpu

SEED = 20250922


def _ng15(kind="full", npsr=None):
    from pta_replicator_b200 import synthetic
    return synthetic.make_ng15_like(kind, npsr=npsr)


def _batch(psrs, noise, gwb=True, tm=True):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise, gwb=gwb)
    if tm:
        for i in range(b.n_psr):
            b.set_timing_model(i, poly=2, jumps="f")
    b.set_optimal_statistic()
    return b


def _numpy_os(b, po, rows):
    """The plan's statics applied with numpy to host rows [R, ld]."""
    nc = po["nc"]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :nc]
                  for i in range(b.n_psr)], axis=1) * np.sqrt(po["phi"])
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    d = np.einsum("rpj,rpj->rp", X[:, pa], X[:, pb])
    bo = d @ po["orf"].T
    return dict(rho=d / po["t_ab"], A2=bo / po["dnorm"], snr=bo / po["dsqrt"], A2_mc=bo @ po["finv"].T)


def test_device_matches_numpy_on_the_same_rows_ng15_full():
    psrs, noise = _ng15()
    b = _batch(psrs, noise)
    po = b.plan()["os"]
    rows = b.generate(64, seed=SEED)                       # post-fit rows (spin + JUMPs)
    got = b.optimal_statistic_of(rows, pairs=True)
    ref = _numpy_os(b, po, rows.cpu().numpy())
    d_rho = float(np.max(np.abs(got["rho"].cpu().numpy() - ref["rho"]) / po["sigma"]))
    d_a2 = float(np.max(np.abs(got["A2"].cpu().numpy() - ref["A2"]) / po["A2_sigma"]))
    d_snr = float(np.max(np.abs(got["snr"].cpu().numpy() - ref["snr"])))
    d_mc = float(np.max(np.abs(got["A2_mc"].cpu().numpy() - ref["A2_mc"]) / np.sqrt(np.diag(po["finv"]))))
    print(f"\n[os] device vs numpy, 64 realizations ng15-full: |drho|/sigma {d_rho:.1e}, |dA2|/A2_sigma {d_a2:.1e}, "
          f"|dS/N| {d_snr:.1e}, |dA2_mc|/sigma_mc {d_mc:.1e}; host statics {po['setup_s']:.1f} s")
    assert d_rho <= 1e-10 and d_a2 <= 1e-10 and d_snr <= 1e-10 and d_mc <= 1e-10
    assert torch_equal(got["sigma"], po["sigma"]) and torch_equal(got["A2_sigma"], po["A2_sigma"])


def torch_equal(t, a):
    return bool(np.array_equal(t.cpu().numpy(), a))


def test_prefit_statistic_equals_postfit_rows():
    """optimal_statistic skips the timing fit: P^{-1} annihilates the timing columns."""
    psrs, noise = _ng15()
    b = _batch(psrs, noise)
    R = 256
    a = b.optimal_statistic(R, seed=SEED, pairs=True)
    c = b.optimal_statistic_of(b.generate(R, seed=SEED), pairs=True)
    d_rho = float((a["rho"] - c["rho"]).abs().div(a["sigma"]).max())
    d_a2 = float((a["A2"] - c["A2"]).abs().div(a["A2_sigma"]).max())
    d_snr = float((a["snr"] - c["snr"]).abs().max())
    print(f"\n[os] pre-fit vs post-fit rows: |drho|/sigma {d_rho:.1e}, |dA2|/A2_sigma {d_a2:.1e}, |dS/N| {d_snr:.1e}; "
          f"max |rho|/sigma {float(a['rho'].abs().div(a['sigma']).max()):.1f}")
    assert max(d_rho, d_a2, d_snr) <= 1e-9


def test_bit_identity_across_chunks_real0_and_paths():
    import torch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise)
    R = 1024
    a = b.optimal_statistic(R, seed=SEED, chunk=1024, pairs=True)
    c = b.optimal_statistic(R, seed=SEED, chunk=256, pairs=True)
    lo = b.optimal_statistic(512, seed=SEED, real0=0, pairs=True)
    hi = b.optimal_statistic(512, seed=SEED, real0=512, pairs=True)
    for k in ("A2", "snr", "A2_mc", "rho"):
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    # without a timing model the generated rows are the rows the statistic reduces
    b2 = _batch(psrs, noise, tm=False)
    e = b2.optimal_statistic(R, seed=SEED, pairs=True)
    f = b2.optimal_statistic_of(b2.generate(R, seed=SEED), pairs=True)
    for k in ("A2", "snr", "A2_mc", "rho"):
        assert torch.equal(e[k], f[k]), k


def test_null_law_ng15_full():
    """White + ECORR + RN with timing models, no GWB, P = the generating model: S/N ~ N(0, 1) per template and
    rho_ab / sigma_ab has unit variance (exact in law)."""
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False)
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 3, pairs=True)
    snr = res["snr"].cpu().numpy()
    z = (res["rho"] / res["sigma"]).cpu().numpy()
    mean, var = snr.mean(axis=0), snr.var(axis=0, ddof=1)
    pooled = z.var()
    # pooled variance of correlated pairs: a 5-sigma bound from the per-pair variance spread
    se = np.sqrt(2.0 / R)
    print(f"\n[os] null law R={R}: S/N mean {np.round(mean, 4)}, var {np.round(var, 4)}; pooled rho/sigma var {pooled:.4f}")
    assert np.all(np.abs(mean) < 4 / np.sqrt(R))
    assert np.all(np.abs(var - 1) < 0.1)
    assert abs(pooled - 1) < 5 * se


def test_injected_gwb_mean_matches_oracle_expectation_ng15_epoch():
    """GWB injected (ng15-epoch, so that the dense oracle fits): mean of A2_HD against the exact E[A2] from the
    injection covariance, within 4 empirical standard errors."""
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=True, tm=True)
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 5)
    a2 = res["A2"].cpu().numpy()[:, 0]
    models = []
    for i, p in enumerate(b.psrs):                          # the oracle's own design matrices, engine order
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        models.append(TO.timing_design_matrix(t, 2, [f.get("f") for f in p.toas.table["flags"]])[b.order[i]])
    S = OO.statics(b, models=models)
    e = OO.expected_a2(b, S)
    A2_inj = 10 ** (2 * -14.6733)
    m, se = a2.mean(), a2.std(ddof=1) / np.sqrt(R)
    print(f"\n[os] signal R={R}: mean A2_HD {m:.4e} +- {se:.1e}, oracle E[A2] {e[0]:.4e}, E[A2]/A2_inj = {e[0] / A2_inj:.4f}")
    assert abs(m - e[0]) < 4 * se
