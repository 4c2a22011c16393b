"""GPU tests of the timing-model fit (``PulsarBatch.set_timing_model`` -> ``ptar_timing_project``): post-fit rows
against the SVD least-squares oracle on the same draws, against the unmodified reference's quadratic removal
(``add_burst(remove_quad=True)``, tests/golden/ref_f4.npz), against the weighted-mean removal of
``simulate.Residuals``, the chi-square law of white noise after the fit, and bit-for-bit reproducibility."""
import os

import numpy as np
import pytest

from tests import timing_oracle as TO
from tests.fixtures import GOLD, load_flags_case, rel_rms

pytestmark = pytest.mark.gpu

SEED = 20250922


def _ng15(npsr=None):
    from pta_replicator_b200 import synthetic
    return synthetic.make_ng15_like("full", npsr=npsr)


def _config2(psrs, noise, white_only=False):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs)
    if white_only:
        for i in range(b.n_psr):
            b.set_white(i, efac=1.0)
    else:
        synthetic.ng15_recipe(b, noise)
    return b


def _oracle_postfit(b, rows, i, poly, jumps=None, extra=None, sigma=None):
    """SVD oracle for pulsar i: rows [R, ld] (engine order) -> post-fit [R, n] in table order."""
    p = b.psrs[i]
    t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
    fv = [f.get(jumps) for f in p.toas.table["flags"]] if jumps else None
    M = TO.timing_design_matrix(t, poly, fv, extra)
    sig = p.toas.get_errors().to("s").value if sigma is None else sigma
    pre = np.stack([b.unpack(r, i) for r in rows])
    return TO.postfit_lstsq(pre, M, sig)


def _annual(p):
    t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
    w = 2 * np.pi / (365.25 * 86400.0)
    return np.stack([np.sin(w * t), np.cos(w * t)], axis=1)


def _worst(b, pre, post, model):
    worst = 0.0
    for i in range(b.n_psr):
        ref = _oracle_postfit(b, pre, i, **model(i))
        got = np.stack([b.unpack(r, i) for r in post])
        worst = max(worst, float(np.max(np.abs(got - ref)) / np.sqrt(np.mean(ref**2))))
    return worst


def test_spin_jumps_against_svd_oracle_same_draws_ng15_full():
    """Config 2 at ng15-full, 8 realizations: pre-fit rows (no model) through the oracle == post-fit rows (spin + JUMPs)."""
    psrs, noise = _ng15()
    b = _config2(psrs, noise)
    pre = b.generate(8, seed=SEED).cpu().numpy()
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    post = b.generate(8, seed=SEED).cpu().numpy()
    worst = _worst(b, pre, post, lambda i: dict(poly=2, jumps="f"))
    print(f"\n[timing] ng15-full spin+jumps, 8 realizations: max|d| / post-fit rms (worst pulsar) = {worst:.2e}")
    assert worst <= 1e-11


def test_linear_plus_annual_sinusoids_against_svd_oracle():
    psrs, noise = _ng15(npsr=4)
    b = _config2(psrs, noise)
    pre = b.generate(8, seed=SEED + 1).cpu().numpy()
    for i, p in enumerate(psrs):
        b.set_timing_model(i, poly=1, extra=_annual(p))
    post = b.generate(8, seed=SEED + 1).cpu().numpy()
    worst = _worst(b, pre, post, lambda i: dict(poly=1, extra=_annual(psrs[i])))
    print(f"\n[timing] poly=1 + annual sin/cos: max|d| / post-fit rms = {worst:.2e}")
    assert worst <= 1e-11


def test_quadratic_fit_matches_reference_remove_quad():
    """The unmodified reference's add_burst(remove_quad=True) (np.polyfit, unweighted) on the 4 flag-case pulsars."""
    import pta_replicator_b200 as api
    from pta_replicator_b200.engine import PulsarBatch
    z = np.load(os.path.join(GOLD, "ref_f4.npz"))
    _, spec = load_flags_case()
    psrs = []
    for s in spec:
        p = api.pulsar_from_arrays(s["name"], s["loc"], s["mjd"].astype(np.longdouble), s["err_us"],
                                   flags=[{"f": f, "pta": "SYN"} for f in s["flag"]])
        api.make_ideal(p)
        psrs.append(p)
    b = PulsarBatch(psrs)
    for i, p in enumerate(psrs):
        b.set_deterministic(i, z[f"burst_{i}"])
        b.set_timing_model(i, poly=2, sigma=np.ones(p.toas.ntoas))
    out = b.generate(4, seed=1).cpu().numpy()
    for i in range(len(psrs)):
        for r in range(4):
            assert rel_rms(b.unpack(out[r], i), z[f"burstq_{i}"]) < 1e-9, (i, r)


def test_offset_fit_equals_simulate_residuals_weighted_mean():
    import pta_replicator_b200 as api
    from pta_replicator_b200 import simulate
    from pta_replicator_b200.engine import PulsarBatch
    psrs = api.load_from_directories(os.path.join(GOLD, "partim_small", "par"), os.path.join(GOLD, "partim_small", "tim"))
    for p in psrs:
        api.make_ideal(p)
    rng = np.random.default_rng(8)
    b = PulsarBatch(psrs)
    delays = []
    for i, p in enumerate(psrs):
        d = 2e-7 + 1e-7 * rng.standard_normal(p.toas.ntoas)
        delays.append(d)
        b.set_deterministic(i, d)
        b.set_timing_model(i, poly=0)
    out = b.generate(4, seed=2).cpu().numpy()
    worst = 0.0
    for i, p in enumerate(psrs):
        T = simulate.TOAs(p.toas.table["tdbld"], p.toas.err_us)
        T.delay_s = delays[i]
        ref = simulate.Residuals(T).time_resids.value
        for r in range(4):
            worst = max(worst, rel_rms(b.unpack(out[r], i), ref))
    print(f"\n[timing] poly=0 vs simulate.Residuals: max|d| / rms = {worst:.2e}")
    assert worst <= 1e-14


def test_white_noise_chi_square_law_after_the_fit():
    """White noise (efac 1, sigma = TOA errors), spin + JUMPs, 4096 realizations at ng15-full: the mean over
    realizations of sum_p sum_i r'^2 / sigma^2 is sum_p (n_p - k_p) within 5 sigma, sigma = sqrt(2 sum (n_p - k_p) / R)."""
    import torch
    psrs, noise = _ng15()
    b = _config2(psrs, noise, white_only=True)
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    tm = b.plan()["tm"]
    idx = np.concatenate([np.arange(b.toa_off[i], b.toa_off[i] + b.ntoa[i]) for i in range(b.n_psr)])
    idx_d = torch.from_numpy(idx).to(b.device)
    w_d = torch.from_numpy(tm["sqrtw"][idx]).to(b.device)
    R, chunk = 4096, 512
    chi2 = []
    for r0 in range(0, R, chunk):
        out = b.generate(chunk, seed=SEED + 7, real0=r0)
        chi2.append(((out[:, idx_d] * w_d) ** 2).sum(dim=1).cpu().numpy())
        del out
    chi2 = np.concatenate(chi2)
    dof = int(sum(b.ntoa) - tm["k"].sum())
    sig = np.sqrt(2.0 * dof / R)
    z = (chi2.mean() - dof) / sig
    z_nofit = (chi2.mean() - sum(b.ntoa)) / sig
    print(f"\n[timing] chi2 law: mean {chi2.mean():.1f}, expected {dof} (sum k_p = {int(tm['k'].sum())}), "
          f"z = {z:.2f}; against sum n_p: z = {z_nofit:.1f}")
    assert abs(z) < 5
    assert abs(z_nofit) > 5


def test_postfit_rows_are_bit_identical_across_chunking_real0_and_host_delivery():
    import torch
    psrs, noise = _ng15(npsr=12)
    b = _config2(psrs, noise)
    for i in range(0, b.n_psr, 2):                 # odd pulsars: no model
        b.set_timing_model(i, poly=2, jumps="f")
    R = 1024
    a = b.generate(R, seed=SEED, chunk=1024)
    c = b.generate(R, seed=SEED, chunk=256)
    assert torch.equal(a, c)
    lo = b.generate(512, seed=SEED, real0=0)
    hi = b.generate(512, seed=SEED, real0=512)
    assert torch.equal(a[:512], lo) and torch.equal(a[512:], hi)
    h = b.generate_to_host(R, seed=SEED, chunk=64)
    assert torch.equal(a.cpu(), h)
    # pulsars without a model and every padding slot are exactly the pre-fit values
    for i in range(0, b.n_psr, 2):
        b.set_timing_model(i, poly=None)           # no column: the model is removed
    pre = b.generate(R, seed=SEED, chunk=1024)
    keep = np.ones(b.ld, dtype=bool)
    for i in range(0, b.n_psr, 2):
        keep[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = False
    keep_d = torch.from_numpy(keep).to(b.device)
    assert torch.equal(a[:, keep_d], pre[:, keep_d])
    assert not torch.equal(a[:, ~keep_d], pre[:, ~keep_d])
