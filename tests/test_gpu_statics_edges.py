"""GPU tests of the chain device -> statics -> definition: the device outputs of edge recipes of
tests/statics_reference.py (``optimal_statistic_of`` with anisotropy and ``aniso_maps``, ``fp_statistic_of`` with the
Fe sky grid and ``maps``, ``curn_likelihood_of`` with HD and ``maps``) against the extended-precision dense reference
of the definitions.  Allowance per output: the statics tolerance of tests/test_statics_edges_cpu.py (relative to the
same scales) plus the rigorous kernel bound of tests/reduction_reference.py on the device's own statics, so one
assertion covers the host statics, their ``compile()`` layout and the kernels.  Pulsars of 5, 7, 65, 193 TOAs; K = 1
and 16."""
import numpy as np
import pytest

from tests import reduction_reference as RR
from tests import statics_reference as SR
from tests.test_statics_edges_cpu import TAU, TAU_LIKE, _kappa, _tau

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _device_batches(monkeypatch):
    monkeypatch.setattr(SR, "PLAN_ONLY", False)


def _t(b, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(b.device)


def _within(dev, ref, allow, what):
    r = float(np.max(np.abs(np.asarray(dev) - ref) / allow))
    print(f"    {what:>14s}: worst |d| / allowance {r:.3g}")
    assert r <= 1.0, f"{what}: |d| / allowance = {r:.3g}"
    return r


def _bound(xref):
    """The kernel bound of a check dict plus the gap between its fp64 head and the exact value."""
    return xref["bound"] + np.abs(xref["lo"])


@pytest.mark.parametrize("name", ["corners_k1", "corners_k16"])
def test_curn_hd_device_against_definition(name):
    from tests.test_gpu_curn_likelihood import _xref as curn_xref
    from tests.test_gpu_hd_likelihood import _xref as hd_xref
    e = SR.recipes()[name]()
    b = e.b
    rows = SR.rows_of(b, 3, seed=len(name))
    res = b.curn_likelihood_of(_t(b, rows), maps=True)
    print(f"\n[statics edges, device] {name}: K = {e.stats['curn']['K']}, TOAs {tuple(b.ntoa)}")
    ref = SR.curn(e, rows)
    xk = curn_xref(b, rows)
    _within(res["lnL"].cpu().numpy(), ref["lnl"], TAU_LIKE * ref["scale"] + _bound(xk),
            "curn lnL")
    if "hd" in e.stats:
        rh = SR.hd(e, rows)
        _within(res["hd_lnL"].cpu().numpy(), rh["lnl"], TAU_LIKE * rh["scale"] + _bound(hd_xref(b, rows)), "hd lnL")


def test_os_and_anisotropy_device_against_definition():
    from tests.test_gpu_reduction_edges import _os_statics
    e = SR.recipes()["aniso_lmax1"]()
    b = e.b
    rows = SR.rows_of(b, 3, seed=7)
    res = b.optimal_statistic_of(_t(b, rows), pairs=True, aniso_maps=True)
    tau = _tau(_kappa(e))
    print(f"\n[statics edges, device] aniso_lmax1: K = {e.stats['os']['K']}, TOAs {tuple(b.ntoa)}")
    Sd = _os_statics(b)
    xo = RR.optimal_statistic(Sd, rows)
    ref = SR.optimal_statistic(e, rows)
    for k in ("rho", "A2", "snr", "A2_mc"):
        _within(res[k].cpu().numpy(), ref[k], tau * ref[k + "_s"] + _bound(xo[k]), "os " + k)
    st = b.compile()["os"]["aniso"]
    am = st["model"]
    N = dict(method="sky_scramble", V=st["dev"]["V"].cpu().numpy().reshape(am.n_colp, am.kdp), kd=am.kd, n_col=am.n_col,
             dsqrt=st["dev"]["dsqrt"].cpu().numpy())
    xa = RR.os_null(Sd, N, xo)["snr"]
    ra = SR.anisotropy(e, rows, b.plan()["os_aniso"]["T_sph"])
    n_lm, n_z = am.n_lm, am.n_z
    _within(res["clm"].cpu().numpy(), ra["clm"], tau * ra["clm_s"] + _bound(xa)[:, :n_lm], "aniso clm")
    zh, zb = xa["hi"][:, n_lm:n_lm + n_z], _bound(xa)[:, n_lm:n_lm + n_z]
    cb = np.sum(2 * np.abs(zh) * zb + zb ** 2, axis=1) + RR.gamma(n_z + 8) * np.sum(zh ** 2, axis=1)
    _within(res["aniso_chi2"].cpu().numpy(), ra["chi2"], tau * (1 + ra["chi2_s"]) + cb, "aniso chi2")
    S = am.n_col - n_lm - n_z
    _within(res["radio_snr"].cpu().numpy(), ra["radio"], tau * ra["radio_s"] + _bound(xa)[:, n_lm + n_z:n_lm + n_z + S],
            "aniso radio")


@pytest.mark.parametrize("name", ["common_loud", "pole_4psr"])
def test_fp_fe_device_against_definition(name):
    from pta_replicator_b200.engine import fp_whitened_basis
    e = SR.recipes()[name]()
    b = e.b
    rows = SR.rows_of(b, 3, seed=len(name))
    res = b.fp_statistic_of(_t(b, rows), pulsars=True, maps=True)
    o = e.stats["fp"]
    kap = _kappa(e)
    if o["log10_A_common"] is not None:
        from tests.test_statics_edges_cpu import _common_fp
        kap = max(SR.woodbury_cond(b, i, _common_fp(e, i), e.tm[i]) for i in range(b.n_psr))
    tau = _tau(kap)
    print(f"\n[statics edges, device] {name}: Nf = {len(o['freqs'])}, TOAs {tuple(b.ntoa)}")
    st = b.compile()["fp"]
    Ct = [fp_whitened_basis(dict(Ct=st["Ct"].cpu().numpy(), n_freq=st["n_freq"]), s, n) for s, n in zip(b.toa_off, b.ntoa)]
    xf = RR.fp_statistic(Ct, b.toa_off, b.ntoa, rows)
    rf = SR.fp(e, rows)
    R, P, Nf = rows.shape[0], b.n_psr, len(o["freqs"])
    ab = _bound(xf["amps"]).reshape(R, P, Nf, 2)
    _within(res["amps"].cpu().numpy(), rf["amps"], tau * np.maximum(1, np.abs(rf["amps"])) + ab, "fp X^")
    _within(res["Fp"].cpu().numpy(), rf["Fp"], tau * rf["Fp"] + _bound(xf["Fp"]), "fp Fp")
    # Fe: the Fp amplitudes' bound through N_a = L_a X^_a, N4 = sum_a e_a (x) N_a and L4^-1, plus the rounding of the
    # combine (gamma_{P+16} on the same absolute sums, gamma_8 on Fe)
    pe = b.plan()["fe"]
    S = pe["n_sky"]
    Lf, ant = pe["Lf"], pe["antenna"]
    Linv = np.zeros(pe["linv"].shape[:2] + (4, 4))
    Linv[..., np.tril_indices(4)[0], np.tril_indices(4)[1]] = pe["linv"]
    X = res["amps"].cpu().numpy()
    l11, l21, l22 = (Lf[None, :, :, j].transpose(0, 2, 1) for j in range(3))
    N = np.stack([l11 * X[..., 0], l21 * X[..., 0] + l22 * X[..., 1]], axis=-1)
    dN = np.stack([np.abs(l11) * ab[..., 0], np.abs(l21) * ab[..., 0] + np.abs(l22) * ab[..., 1]], axis=-1)
    yabs = np.abs(np.einsum("fsij,rfsj->rfsi", Linv[:, :S],
                            np.einsum("asp,rafc->rfspc", ant, N).reshape(R, Nf, S, 4)))
    t = np.einsum("fsij,rfsj->rfsi", np.abs(Linv[:, :S]),
                  np.einsum("asp,rafc->rfspc", np.abs(ant), np.abs(N)).reshape(R, Nf, S, 4))
    d = np.einsum("fsij,rfsj->rfsi", np.abs(Linv[:, :S]),
                  np.einsum("asp,rafc->rfspc", np.abs(ant), dN).reshape(R, Nf, S, 4))
    Fe = res["Fe"].cpu().numpy()
    fb = np.sum(yabs * (d + RR.gamma(P + 16) * t) + d * d, axis=-1) + RR.gamma(8) * Fe
    rfe = SR.fe(e, rows, rf)
    _within(Fe, rfe["Fe"], tau * np.maximum(1, rf["Fp"])[:, :, None] + fb, "fe Fe")
