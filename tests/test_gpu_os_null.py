"""GPU tests of the optimal statistic's null distributions (``PulsarBatch.set_os_null`` -> ``ptar_os_null``), both
methods: the device against the plan's statics applied in numpy on the same rows, bit-identity across chunking, real0
splits and paths, the exact null law without a GWB, and the injected-signal mean of every column against the dense
oracle's exact expectation."""
import numpy as np
import pytest

from tests import os_null_oracle as NO
from tests import os_oracle as OO
from tests import timing_oracle as TO
from tests.test_gpu_optimal_statistic import SEED, _batch, _ng15

pytestmark = pytest.mark.gpu

METHODS = ["phase_shift", "sky_scramble"]


def _u(b, po, rows, method):
    """ptar_os_null's U [R, kd] from host rows, with the plan's C."""
    nc = po["nc"]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :nc]
                  for i in range(b.n_psr)], axis=1) * np.sqrt(po["phi"])
    xa, xb = X[:, po["pairs"][:, 0]], X[:, po["pairs"][:, 1]]
    if method == "sky_scramble":
        return np.einsum("rqj,rqj->rq", xa, xb)
    sa, ca, sb, cb = xa[..., 0::2], xa[..., 1::2], xb[..., 0::2], xb[..., 1::2]
    return np.stack([sa * sb + ca * cb, ca * sb - sa * cb], axis=-1).reshape(len(rows), -1)


@pytest.mark.parametrize("method", METHODS)
def test_device_matches_plan_statics_ng15_full(method):
    psrs, noise = _ng15()
    b = _batch(psrs, noise)
    n = 200                                                   # 201 columns: four column blocks, the last one partial
    b.set_os_null(method, n=n, seed=11)
    pl = b.plan()
    po, pn = pl["os"], pl["os_null"]
    rows = b.generate(64, seed=SEED)
    got = b.optimal_statistic_of(rows, null_values=True)
    ref = _u(b, po, rows.cpu().numpy(), method) @ pn["V"][:n + 1, :pn["kd"]].T / pn["dsqrt"]
    ns = got["null_snr"].cpu().numpy()
    d = float(np.max(np.abs(ns - ref)))
    d0 = float(np.max(np.abs(ns[:, 0] - got["snr"][:, 0].cpu().numpy())))
    print(f"\n[os null] {method} device vs numpy, 64 ng15-full rows x {n + 1} columns: |dS/N| {d:.1e}; column 0 vs "
          f"os_pairs {d0:.1e}; null statics {pn['setup_s']:.2f} s")
    assert d <= 1e-10 and d0 <= 1e-10
    cnt = (ns[:, 1:] >= ns[:, :1]).sum(axis=1)
    assert np.array_equal(got["null_exceed"].cpu().numpy(), cnt)
    assert np.array_equal(got["fap"].cpu().numpy(), (1.0 + cnt) / (n + 1))
    assert got["null_method"] == method and got["null_template"] == "hd"
    assert np.array_equal(got["null_dsqrt"].cpu().numpy(), pn["dsqrt"])
    key = "null_phases" if method == "phase_shift" else "null_radec"
    assert np.array_equal(got[key].cpu().numpy(), pn["phases" if method == "phase_shift" else "radec"])


@pytest.mark.parametrize("method", METHODS)
def test_bit_identity_across_chunks_real0_and_paths(method):
    import torch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise)
    b.set_os_null(method, n=100, seed=2)
    R = 1024
    keys = ("null_snr", "null_exceed", "fap", "snr")
    a = b.optimal_statistic(R, seed=SEED, chunk=1024, null_values=True)
    c = b.optimal_statistic(R, seed=SEED, chunk=256, null_values=True)
    lo = b.optimal_statistic(512, seed=SEED, real0=0, null_values=True)
    hi = b.optimal_statistic(512, seed=SEED, real0=512, null_values=True)
    for k in keys:
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    # without null_values the counts come from the scratch S/N and are the same
    assert torch.equal(b.optimal_statistic(R, seed=SEED, chunk=256)["null_exceed"], a["null_exceed"])
    b2 = _batch(psrs, noise, tm=False)
    b2.set_os_null(method, n=100, seed=2)
    e = b2.optimal_statistic(R, seed=SEED, null_values=True)
    f = b2.optimal_statistic_of(b2.generate(R, seed=SEED), null_values=True)
    for k in keys:
        assert torch.equal(e[k], f[k]), k


@pytest.mark.parametrize("method", METHODS)
def test_exact_null_law_ng15_full(method):
    """No GWB, P = the generating model: every column of the null is N(0, 1) in law (phase shifts: only with the shifted
    t'_ab in D_s); for scrambles, corr(S/N_0, S/N_s) = sum_q G_q G^s_q t_q / sqrt(D_0 D_s)."""
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False)
    b.set_os_null(method, n=64, seed=7)
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 3, null_values=True)
    ns = res["null_snr"].cpu().numpy()
    mean, var = ns.mean(axis=0), ns.var(axis=0, ddof=1)
    print(f"\n[os null] {method} null law R={R}, 65 columns: |mean| <= {np.abs(mean).max():.4f}, var {var.min():.4f}.."
          f"{var.max():.4f}; mean p-value {float(res['fap'].mean()):.4f}")
    assert np.all(np.abs(mean) < 4 / np.sqrt(R))
    assert np.all(np.abs(var - 1) < 0.1)
    if method == "sky_scramble":
        pl = b.plan()
        po, pn = pl["os"], pl["os_null"]
        V = pn["V"][:65, :pn["kd"]]
        pred = (V[0] * V) @ po["t_ab"] / (pn["dsqrt"][0] * pn["dsqrt"])
        emp = np.array([np.corrcoef(ns[:, 0], ns[:, s])[0, 1] for s in range(65)])
        print(f"[os null] scramble correlations: predicted |corr| <= {np.abs(pred[1:]).max():.3f}, "
              f"max |emp - pred| = {np.abs(emp - pred)[1:].max():.4f}")
        assert np.all(np.abs(emp - pred)[1:] < 5 / np.sqrt(R))


@pytest.mark.parametrize("method", METHODS)
def test_injected_gwb_mean_matches_oracle_expectation_ng15_epoch(method):
    """GWB injected (ng15-epoch, so that the dense oracle fits): mean S/N of every column against the exact E[S/N_s]
    = E[A2_s] sqrt(D_s), the oracle's statics rebuilt with the shifted basis or the scrambled template."""
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=True, tm=True)
    n = 8
    b.set_os_null(method, n=n, seed=13)
    R = 4096
    res = b.optimal_statistic(R, seed=SEED + 5, null_values=True)
    ns = res["null_snr"].cpu().numpy()
    models = []
    for i, p in enumerate(b.psrs):
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        models.append(TO.timing_design_matrix(t, 2, [f.get("f") for f in p.toas.table["flags"]])[b.order[i]])
    S0 = OO.statics(b, models=models, templates=("hd",))
    exp = np.empty(n + 1)
    for s in range(n + 1):
        if s == 0:
            S = S0
        elif method == "phase_shift":
            S = NO.phase_shifted_statics(b, res["null_phases"][s - 1].cpu().numpy(), models=models, templates=("hd",))
        else:
            S = NO.scrambled_statics(S0, res["null_radec"][s - 1].cpu().numpy(), "hd")
        exp[s] = OO.expected_a2(b, S)[0] * np.sqrt(S["D"][0])
    m, se = ns.mean(axis=0), ns.std(axis=0, ddof=1) / np.sqrt(R)
    z = (m - exp) / se
    print(f"\n[os null] {method} signal R={R}: E[S/N] column 0 {exp[0]:.3f}, columns 1.. {np.round(exp[1:], 3)}; "
          f"(mean - E) / se {np.round(z, 2)}")
    assert np.all(np.abs(z) < 4)
