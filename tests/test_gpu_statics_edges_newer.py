"""GPU tests of the chain device -> statics -> definition at the chromatic and red-noise edge recipes of
tests/statics_reference.py: ``red_noise_likelihood_of``, ``curn_likelihood_of`` with HD and ``optimal_statistic_of``
with its per-frequency outputs against the extended-precision dense reference of the definitions, DM and scattering noise in every P_a.  Allowance
per output, as in tests/test_gpu_statics_edges.py: the statics tolerance of the CPU tests (relative to the same
scales) plus the rigorous kernel bound of tests/reduction_reference.py on the device's own statics."""
import numpy as np
import pytest

from tests import reduction_reference as RR
from tests import statics_reference as SR
from tests.test_gpu_statics_edges import _bound, _t, _within
from tests.test_statics_edges_cpu import TAU_LIKE, _kappa, _tau

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _device_batches(monkeypatch):
    monkeypatch.setattr(SR, "PLAN_ONLY", False)


@pytest.mark.parametrize("name", ["chrom_all", "chrom_dm_only_rn", "rn_short_span"])
def test_rn_device_against_definition(name):
    from tests.test_gpu_red_noise_likelihood import _xref
    e = SR.recipes()[name]()
    b = e.b
    rows = SR.rows_of(b, 3, seed=len(name))
    res = b.red_noise_likelihood_of(_t(b, rows), maps=True)
    print(f"\n[statics edges, device] {name}: rn K = {e.stats['rn']['K']}, TOAs {tuple(b.ntoa)}")
    ref = SR.rn(e, rows)
    _within(res["lnL"].cpu().numpy(), ref["lnl"], TAU_LIKE * ref["scale"] + _bound(_xref(b, rows)), "rn lnL")


@pytest.mark.parametrize("name", ["chrom_all", "chrom_single_freq"])
def test_curn_hd_os_device_on_chromatic_recipes(name):
    from tests.test_gpu_curn_likelihood import _xref as curn_xref
    from tests.test_gpu_hd_likelihood import _xref as hd_xref
    from tests.test_gpu_reduction_edges import _os_statics
    e = SR.recipes()[name]()
    b = e.b
    rows = SR.rows_of(b, 3, seed=len(name))
    print(f"\n[statics edges, device] {name}: K = {e.stats['curn']['K']}, TOAs {tuple(b.ntoa)}")
    res = b.curn_likelihood_of(_t(b, rows), maps=True)
    ref = SR.curn(e, rows)
    _within(res["lnL"].cpu().numpy(), ref["lnl"], TAU_LIKE * ref["scale"] + _bound(curn_xref(b, rows)), "curn lnL")
    if "hd" in e.stats:
        rh = SR.hd(e, rows)
        _within(res["hd_lnL"].cpu().numpy(), rh["lnl"], TAU_LIKE * rh["scale"] + _bound(hd_xref(b, rows)), "hd lnL")
    tau = _tau(_kappa(e))
    ro = b.optimal_statistic_of(_t(b, rows), pairs=True)
    xo = RR.optimal_statistic(_os_statics(b), rows)
    rf = SR.optimal_statistic(e, rows)
    for k in ("rho", "A2", "snr", "A2_mc"):
        _within(ro[k].cpu().numpy(), rf[k], tau * rf[k + "_s"] + _bound(xo[k]), "os " + k)
    if e.stats["os"].get("pf"):
        _check_pfos(e, rows, ro, tau)


def _check_pfos(e, rows, res, tau):
    """The per-frequency outputs against the definition (``SR.pfos``).  Kernel bound on the device's statics: the
    projection's bound (``RR.projection``, with the gap between its fp64 head and the exact value) carried through
    d_qk = X_a,k . X_b,k and the template sums, plus twice the rounding bound of ``_pf_longdouble`` (gamma_3 on d,
    gamma_{n+2} sum |Gamma| (|X_s X_s| + |X_c X_c|) on b, gamma_5 through F_k^-1) evaluated at the exact projection."""
    from tests.test_gpu_os_per_frequency import _pf_longdouble
    from tests.test_gpu_reduction_edges import _os_statics
    b = e.b
    pl = b.plan()
    po, pp = pl["os"], pl["os_pf"]
    Cd, nc = _os_statics(b)["C"], po["nc"]
    R, P, K = rows.shape[0], b.n_psr, pp["K"]
    Xh, XB = np.zeros((R, P, nc)), np.zeros((R, P, nc))
    for a in range(P):
        h, lo, bd, _ = RR.projection(rows, Cd[:, :nc], b.toa_off[a], b.ntoa[a])
        Xh[:, a], XB[:, a] = h, bd + np.abs(lo.astype(np.float64))
    ref = _pf_longdouble(po, pp, Xh)
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    A = np.abs(Xh)
    dB = (A[:, pa] * XB[:, pb] + XB[:, pa] * A[:, pb] + XB[:, pa] * XB[:, pb]).reshape(R, len(pa), K, 2).sum(axis=3)
    dB = dB.transpose(0, 2, 1)                                                       # [R, K, q]
    bB = np.einsum("oq,rkq->rok", np.abs(po["orf"]), dB)
    prop = dict(pf_rho=dB / pp["t"], pf_phi=bB / pp["dnorm"], pf_snr=bB / pp["dsqrt"],
                pf_phi_mc=np.einsum("kop,rpk->rok", np.abs(pp["finv"]), bB))
    rf = SR.pfos(e, rows)
    for k, key in (("pf_rho", "rho"), ("pf_phi", "phi"), ("pf_snr", "snr"), ("pf_phi_mc", "phi_mc")):
        kb = prop[k] + 2 * ref[k][1].astype(np.float64)      # |device - exact evaluation on the device's statics|
        _within(res[k].cpu().numpy(), rf[key], tau * rf[key + "_s"] + kb, "pfos " + key)
