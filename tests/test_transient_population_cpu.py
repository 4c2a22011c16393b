"""Transient populations on the host: the Philox uniform streams of kinds 9 and 10 (tests/tpop_oracle.py) against
Philox4x32-10 itself and against the other streams, the draw transform's laws (KS tests), the per-pulsar coefficients
against ``antenna_patterns`` and the ``add_gw_memory`` / ``add_burst`` formulas, the argument checks of
``set_bwm_population`` and ``set_burst_population`` on a plan-only batch, and the new kernels' ptxas resources."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
from scipy import stats

from oracle.philox import philox4x32_10
from tests import cwpop_oracle as CO
from tests import generator_reference as GR
from tests import tpop_oracle as TO

SEED = 0x1234ABCD5678


def _batch(ntoas=(7, 33, 64)):
    from pta_replicator_b200.engine import PulsarBatch
    return PulsarBatch(GR.dense_pulsars(ntoas, seed=11, name="P"), plan_only=True)


def _span(b):
    return min(float(m.min()) for m in b.mjd), max(float(m.max()) for m in b.mjd)


def _phat(b):
    from pta_replicator_b200 import orf
    locs = orf.psrlocs_from_pulsars(b.psrs)
    th, ph = np.pi / 2 - locs[:, 1], locs[:, 0]
    return th, ph, np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], axis=1)


# ------------------------------------------------------------------ the uniform streams
@pytest.mark.parametrize("kind", (TO.K_BWMPOP, TO.K_BURSTPOP))
def test_words_are_philox_at_the_documented_counters(kind):
    elem = np.array([0, 1, 2, 4, 16 * 5 + 3, 16 * 63 + 4])
    for r in (0, 1, 7, 2**32 + 5):
        w = TO.words(kind, elem, r, SEED)
        ref = philox4x32_10(elem, kind, r & 0xFFFFFFFF, r >> 32, SEED)
        for a, b in zip(w, ref):
            assert np.array_equal(a, b)
        u = TO.uniforms(kind, elem, r, SEED)
        assert np.array_equal(u[:, 0], CO.uniform53(ref[0], ref[1]))
        assert np.array_equal(u[:, 1], CO.uniform53(ref[2], ref[3]))


def _blocks(w):
    a = np.ascontiguousarray(np.stack([x.ravel() for x in w], axis=1).astype(np.uint32))
    return a.view(np.dtype((np.void, 16))).ravel()


def test_no_collision_with_other_streams_or_between_families():
    elem = np.arange(64 * 16)
    r = np.arange(64)[:, None]
    bwm, burst = _blocks(TO.words(TO.K_BWMPOP, elem, r, SEED)), _blocks(TO.words(TO.K_BURSTPOP, elem, r, SEED))
    assert np.unique(bwm).size == bwm.size and np.unique(burst).size == burst.size
    assert np.intersect1d(bwm, burst).size == 0
    for kind in range(1, 9):
        for rf in (r, r >> 2):          # the noise streams key (c.z, c.w) on r >> 2, the populations on r
            for psr in (0, 1, 66):
                w = _blocks(philox4x32_10(elem, kind | (psr << 8), rf, 0, SEED))
                assert np.intersect1d(bwm, w).size == 0 and np.intersect1d(burst, w).size == 0, (kind, psr)


# ------------------------------------------------------------------ the draw transform
def test_bwm_laws_ks():
    b = _batch()
    b.set_bwm_population(n_sources=2)
    d = TO.draw(b._bwmpop, np.arange(50_000), SEED)
    first, last = _span(b)
    laws = dict(t0=(d[..., TO.T0] - first) / (last - first), log10_strain=(d[..., TO.LOG10_AMP] + 15) / 3,
                gwtheta=(np.cos(d[..., TO.GWTHETA]) + 1) / 2, gwphi=d[..., TO.GWPHI] / (2 * np.pi),
                bwm_pol=d[..., TO.POL] / np.pi)
    for name, x in laws.items():
        assert stats.kstest(x.ravel(), "uniform").pvalue > 1e-3, name
    assert np.all(d[..., 5:] == 0.0)
    assert abs(stats.pearsonr(laws["t0"].ravel(), laws["log10_strain"].ravel())[0]) < 0.02


def test_burst_laws_ks():
    b = _batch()
    b.set_burst_population(n_sources=2)
    d = TO.draw(b._burstpop, np.arange(50_000), SEED)
    first, last = _span(b)
    Tspan = b._array_tspan(None)
    f0 = 10.0 ** d[..., TO.LOG10_F0]
    assert f0.min() >= 2 / Tspan * (1 - 1e-12) and f0.max() <= 20 / Tspan * (1 + 1e-12)
    laws = dict(t0=(d[..., TO.T0] - first) / (last - first), log10_amp=(d[..., TO.LOG10_AMP] + 8) / 2,
                log10_f0=np.log(f0 * Tspan / 2) / np.log(10.0), Q=(d[..., TO.Q] - 4) / 4,
                gwtheta=(np.cos(d[..., TO.GWTHETA]) + 1) / 2, gwphi=d[..., TO.GWPHI] / (2 * np.pi),
                psi=d[..., TO.POL] / np.pi, phase0=d[..., TO.PHASE0] / (2 * np.pi), eps=d[..., TO.EPS])
    for name, x in laws.items():
        assert stats.kstest(x.ravel(), "uniform").pvalue > 1e-3, name
    assert np.all(d[..., 9] == 0.0)
    for a, c in (("t0", "log10_f0"), ("gwtheta", "psi"), ("Q", "eps")):
        assert abs(stats.pearsonr(laws[a].ravel(), laws[c].ravel())[0]) < 0.02, (a, c)


def test_fixed_and_ranged_parameters():
    b = _batch()
    b.set_burst_population(n_sources=3, log10_amp=-7.25, t0_mjd=(53100.0, 53200.0), log10_f0=-8.5, Q=5.0, gwtheta=1.1,
                           gwphi=0.3, psi=(0.2, 0.4), phase0=2.0, eps=0.5)
    d = TO.draw(b._burstpop, np.arange(4096), SEED)
    for j, v in ((TO.LOG10_AMP, -7.25), (TO.LOG10_F0, -8.5), (TO.Q, 5.0), (TO.GWTHETA, 1.1), (TO.GWPHI, 0.3),
                 (TO.PHASE0, 2.0), (TO.EPS, 0.5)):
        assert np.all(d[..., j] == v), j
    assert d[..., TO.T0].min() >= 53100.0 and d[..., TO.T0].max() < 53200.0
    assert d[..., TO.POL].min() >= 0.2 and d[..., TO.POL].max() < 0.4


# ------------------------------------------------------------------ coefficients against the drop-ins' formulas
def test_patterns_equal_antenna_patterns():
    from pta_replicator_b200.engine import antenna_patterns
    b = _batch()
    th, ph, phat = _phat(b)
    rng = np.random.default_rng(3)
    sky = np.stack([np.arccos(rng.uniform(-1, 1, 200)), rng.uniform(0, 2 * np.pi, 200)], axis=1)
    ref = antenna_patterns(th, ph, sky)
    for k in range(len(sky)):
        np.testing.assert_allclose(TO.patterns(phat, *sky[k]), ref[:, k], rtol=1e-12, atol=1e-14)
    # on a pulsar's line of sight and antipodal to it: (0, 0), as antenna_patterns
    for gt, gp in ((th[1], ph[1]), (np.pi - th[1], (ph[1] + np.pi) % (2 * np.pi))):
        F = TO.patterns(phat, gt, gp)
        assert np.all(np.isfinite(F)) and F[1, 0] == 0.0 and F[1, 1] == 0.0


def test_bwm_coefficient_is_add_gw_memory_polarisation():
    from pta_replicator_b200.deterministic import _antenna
    b = _batch()
    _, _, phat = _phat(b)
    b.set_bwm_population(n_sources=4)
    d = TO.draw(b._bwmpop, np.arange(16), SEED)
    for v in d.reshape(-1, TO.NPAR):
        c = TO.coefficients(TO.BWM, v, phat)
        for a, p in enumerate(b.psrs):
            fp, fx = _antenna(p, v[TO.GWTHETA], v[TO.GWPHI])
            pol = np.cos(2 * v[TO.POL]) * fp + np.sin(2 * v[TO.POL]) * fx
            np.testing.assert_allclose(c[a, 0], pol * 10.0 ** v[TO.LOG10_AMP], rtol=1e-9, atol=1e-12 * 10.0 ** v[TO.LOG10_AMP])
        assert np.all(c[:, 1] == 0.0)


def test_burst_coefficients_against_add_burst():
    """alpha, beta: ``add_burst``'s rotation and projection (burst_kernel) of the restated waveforms equal
    g (alpha cos Phi + beta sin Phi); a1..a4: the rotated polarisations equal the search's waveforms at psi = 0."""
    from pta_replicator_b200.deterministic import _antenna
    b = _batch()
    _, _, phat = _phat(b)
    b.set_burst_population(n_sources=3)
    d = TO.draw(b._burstpop, np.arange(12), SEED)
    t = np.linspace(*_span(b), 2000) * 86400.0
    for v in d.reshape(-1, TO.NPAR):
        hp, hx = TO.waveforms(v, t)
        c2, s2 = np.cos(2 * v[TO.POL]), np.sin(2 * v[TO.POL])
        rplus, rcross = hp * c2 - hx * s2, hp * s2 + hx * c2
        f0 = 10.0 ** v[TO.LOG10_F0]
        dt = t - v[TO.T0] * 86400.0
        g = np.exp(-(dt * 2 * np.pi * f0 / v[TO.Q]) ** 2)
        ph, x = 2 * np.pi * f0 * dt + v[TO.PHASE0], 2 * np.pi * f0 * dt
        A = 10.0 ** v[TO.LOG10_AMP]
        co = TO.coefficients(TO.BURST, v, phat)
        for a, p in enumerate(b.psrs):
            fp, fx = _antenna(p, v[TO.GWTHETA], v[TO.GWPHI])
            res = -fp * rplus - fx * rcross
            np.testing.assert_allclose(g * (co[a, 0] * np.cos(ph) + co[a, 1] * np.sin(ph)), res, rtol=0, atol=1e-9 * A)
        a1, a2, a3, a4 = TO.search_amplitudes(v)
        np.testing.assert_allclose(a1 * g * np.cos(x) + a2 * g * np.sin(x), rplus, rtol=0, atol=1e-12 * A)
        np.testing.assert_allclose(a3 * g * np.cos(x) + a4 * g * np.sin(x), rcross, rtol=0, atol=1e-12 * A)


# ------------------------------------------------------------------ registration
def test_registration_and_removal():
    from pta_replicator_b200.engine import PulsarBatch
    b = _batch()
    assert b._bwmpop is None and b._burstpop is None
    b._compiled = "x"
    b.set_bwm_population(n_sources=2, log10_strain=-13.0, t0_mjd=53005.0)
    assert b._compiled is None
    p = b._bwmpop
    assert p["family"] == TO.BWM and p["n_src"] == 2 and len(p["kind"]) == TO.NPAR
    assert p["kind"][:5] == [CO.FIXED, CO.FIXED, CO.ACOS, CO.UNIFORM, CO.UNIFORM] and p["lo"][0] == 53005.0
    b.set_burst_population()
    p = b._burstpop
    first, last = _span(b)
    Tspan = b._array_tspan(None)
    assert p["family"] == TO.BURST and p["lo"][TO.T0] == first and p["width"][TO.T0] == last - first
    assert p["lo"][TO.LOG10_F0] == np.log10(2 / Tspan)
    assert p["width"][TO.LOG10_F0] == np.log10(20 / Tspan) - np.log10(2 / Tspan)
    assert [k for k, _, _ in (PulsarBatch.CWPOP_ANGLES[n][1] for n in ("psi", "phase0"))] == [CO.UNIFORM, CO.UNIFORM]
    assert b._bwmpop is not None                         # both registered at once
    b._compiled = "x"
    b.set_bwm_population(None)
    b.set_burst_population(None)
    assert b._bwmpop is None and b._burstpop is None and b._compiled is None


@pytest.mark.parametrize("kw", [
    dict(log10_strain=(-12.0, -15.0)), dict(log10_strain=float("nan")), dict(log10_strain=400.0), dict(log10_strain=None),
    dict(t0_mjd=-1.0), dict(t0_mjd=(53000.0, 2e6)), dict(t0_mjd=(53000.0, 53000.0)), dict(t0_mjd="x"),
    dict(gwtheta=-0.1), dict(gwphi=6.3), dict(bwm_pol=3.2), dict(bwm_pol=(0.0, 4.0)), dict(bwm_pol=float("inf")),
    dict(n_sources=0), dict(n_sources=65), dict(n_sources=1.5),
])
def test_bwm_bad_arguments_raise(kw):
    b = _batch()
    with pytest.raises(ValueError):
        b.set_bwm_population(**kw)
    assert b._bwmpop is None


@pytest.mark.parametrize("kw", [
    dict(log10_amp=(-6.0, -8.0)), dict(log10_amp=None), dict(log10_amp=(1, 2, 3)), dict(t0_mjd=2e6),
    dict(log10_f0=(-7.0, float("inf"))), dict(log10_f0=-301.0), dict(Q=0.0), dict(Q=(-1.0, 4.0)), dict(Q=2e6),
    dict(Q=None), dict(eps=1.5), dict(eps=(-0.1, 1.0)), dict(eps=None), dict(psi=3.2), dict(phase0=(-1.0, 1.0)),
    dict(gwtheta=(0.0, 3.2)), dict(n_sources=0), dict(n_sources=65), dict(n_sources=True),
])
def test_burst_bad_arguments_raise(kw):
    b = _batch()
    with pytest.raises(ValueError):
        b.set_burst_population(**kw)
    assert b._burstpop is None


def test_plan_only_device_calls_raise():
    from pta_replicator_b200 import _cabi
    b = _batch()
    b.set_bwm_population(n_sources=2)
    b.set_burst_population(n_sources=2)
    b.plan()
    for fn in (b.bwm_population_params, b.burst_population_params, b.generate):
        with pytest.raises(_cabi.PtarError):
            fn(8)


# ------------------------------------------------------------------ ptxas resources
def test_kernels_have_no_spills():
    from __graft_entry__ import CSRC, NVCC_FLAGS, _nvcc
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_nvcc()] + NVCC_FLAGS + ["-Xptxas", "-v", "-o", os.path.join(d, "lib.so"),
                                                   os.path.join(CSRC, "ptar.cu")], cwd=d, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    found = 0
    for name in ("tpop_draw_kernel", r"tpop_add_kernelILi0E", r"tpop_add_kernelILi1E"):
        m = re.search(name + r"[^\n]*'[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", text)
        assert m, name
        assert m.groups()[1:] == ("0", "0"), (name, m.groups())
        found += 1
    assert found == 3
