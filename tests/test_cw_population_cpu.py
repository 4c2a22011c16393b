"""Continuous-wave populations on the host: the Philox uniform stream of kind 7 (tests/cwpop_oracle.py) against
Philox4x32-10 itself, the draw transform's laws (KS tests), the per-source and per-pulsar constants against
``PulsarBatch.cgw_inputs`` and the argument checks of ``set_cw_population`` on a plan-only batch."""
import numpy as np
import pytest
from scipy import stats

from oracle.philox import philox4x32_10
from tests import cwpop_oracle as CO
from tests import generator_reference as GR

SEED = 0x1234ABCD5678


def _batch(ntoas=(7, 33, 64), **kw):
    from pta_replicator_b200.engine import PulsarBatch
    return PulsarBatch(GR.dense_pulsars(ntoas, seed=11, name="P"), plan_only=True, **kw)


# ------------------------------------------------------------------ the uniform stream
def test_words_are_philox_at_the_documented_counters():
    elem = np.array([0, 1, 3, 4, 16 * 5 + 2, 16 * 63 + 4])
    for psr in (0, 1, 66):
        for r in (0, 1, 7, 2**32 + 5):
            w = CO.words(elem, psr, r, SEED)
            ref = philox4x32_10(elem, 7 | (psr << 8), r & 0xFFFFFFFF, r >> 32, SEED)
            for a, b in zip(w, ref):
                assert np.array_equal(a, b)
            u = CO.uniforms53(elem, psr, r, SEED)
            a = (ref[0].astype(np.uint64) >> np.uint64(5)).astype(float) * 2.0 ** 26 + (ref[1] >> 6).astype(float)
            assert np.array_equal(u[:, 0], a * 2.0 ** -53)


def test_uniforms_in_unit_interval():
    assert CO.uniform53(0, 0) == 0.0
    top = CO.uniform53(0xFFFFFFFF, 0xFFFFFFFF)
    assert top < 1.0 and top == 1.0 - 2.0 ** -53
    u = CO.uniforms53(np.arange(4096), 0, np.arange(4096)[:, None], SEED)
    assert u.min() >= 0.0 and u.max() < 1.0
    assert np.all(u * 2.0 ** 53 == np.floor(u * 2.0 ** 53))                      # 53-bit grid


def test_streams_do_not_coincide():
    base = CO.uniforms53(np.arange(64), 0, np.arange(256)[:, None], SEED).ravel()
    assert np.unique(base).size == base.size                                      # sources x slots x realizations
    others = [CO.uniforms53(np.arange(64), 3, np.arange(256)[:, None], SEED).ravel(),     # another pulsar
              CO.uniforms53(np.arange(64), 0, np.arange(256)[:, None] + 2**32, SEED).ravel(),   # high realization word
              CO.uniforms53(np.arange(64), 0, np.arange(256)[:, None], SEED + 1).ravel()]       # another seed
    for o in others:
        assert np.intersect1d(base, o).size == 0


def _blocks(w):
    """The 128-bit outputs of Philox calls (4 words each) as one comparable key per call."""
    a = np.ascontiguousarray(np.stack([x.ravel() for x in w], axis=1).astype(np.uint32))
    return a.view(np.dtype((np.void, 16))).ravel()


def test_no_collision_with_noise_kinds():
    elem = np.arange(512)
    r = np.arange(64)[:, None]
    mine = _blocks(CO.words(elem, 0, r, SEED))
    for kind in range(1, 7):
        for rf in (r, r >> 2):          # the noise streams key (c.z, c.w) on r >> 2
            w = _blocks(philox4x32_10(elem, kind, rf, 0, SEED))
            assert np.intersect1d(mine, w).size == 0, kind


# ------------------------------------------------------------------ the draw transform
def _pop(b):
    return b._cwpop


def test_draw_laws_ks():
    b = _batch()
    b.set_cw_population(n_sources=1, log10_h0=(-15.0, -13.0), log10_fgw=(-8.7, -7.3), log10_mc=(8.0, 10.0))
    d = CO.draw(_pop(b), np.arange(100_000), SEED)
    laws = dict(gwtheta=(np.cos(d["gwtheta"]) + 1) / 2, gwphi=d["gwphi"] / (2 * np.pi), phase0=d["phase0"] / (2 * np.pi),
                psi=d["psi"] / np.pi, inc=(np.cos(d["inc"]) + 1) / 2, log10_h0=(d["log10_h0"] + 15) / 2,
                log10_fgw=(d["log10_fgw"] + 8.7) / 1.4, log10_mc=(d["log10_mc"] - 8) / 2)
    for name, x in laws.items():
        p = stats.kstest(x.ravel(), "uniform").pvalue
        assert p > 1e-3, (name, p)
    for a, c in (("gwtheta", "inc"), ("gwphi", "psi"), ("log10_h0", "phase0")):   # independent pairs
        assert abs(stats.pearsonr(laws[a].ravel(), laws[c].ravel())[0]) < 0.02, (a, c)


def test_fixed_parameters_exact():
    b = _batch()
    b.set_cw_population(n_sources=3, log10_h0=-14.123456789, log10_fgw=-8.0, log10_mc=9.5, gwtheta=1.1, gwphi=0.3,
                        phase0=2.0, psi=0.7, inc=0.4)
    d = CO.draw(_pop(b), np.arange(64), SEED)
    for name, v in dict(log10_h0=-14.123456789, log10_fgw=-8.0, log10_mc=9.5, gwtheta=1.1, gwphi=0.3, phase0=2.0,
                        psi=0.7, inc=0.4).items():
        assert np.all(d[name] == v), name


def test_ranged_angle_is_uniform_in_the_angle():
    b = _batch()
    b.set_cw_population(gwtheta=(0.2, 0.9), inc=(0.0, 0.5))
    d = CO.draw(_pop(b), np.arange(20_000), SEED)
    assert d["gwtheta"].min() >= 0.2 and d["gwtheta"].max() < 0.9
    assert stats.kstest((d["gwtheta"].ravel() - 0.2) / 0.7, "uniform").pvalue > 1e-3
    assert stats.kstest(d["inc"].ravel() / 0.5, "uniform").pvalue > 1e-3


# ------------------------------------------------------------------ constants against cgw_inputs
@pytest.mark.parametrize("pphase", (None, "uniform"))
def test_constants_equal_cgw_inputs(pphase):
    b = _batch()
    pdist = np.array([0.5, 1.3, 2.0])
    b.set_cw_population(n_sources=3, log10_mc=(8.5, 9.5), pdist=pdist, pphase=pphase)
    d = CO.draw(_pop(b), np.arange(40), SEED, b.n_psr)
    from pta_replicator_b200 import orf
    locs = orf.psrlocs_from_pulsars(b.psrs)
    th, ph = np.pi / 2 - locs[:, 1], locs[:, 0]
    phat = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], axis=1)
    for r in range(40):
        for s in range(3):
            g = {k: float(d[k][r, s]) for k in ("gwtheta", "gwphi", "phase0", "psi", "inc", "fgw", "mc", "h0")}
            dist = CO.dist_mpc(g["h0"], g["fgw"], g["mc"])
            pph = None if pphase is None else d["pphase"][r, s]
            a = b.cgw_inputs(g["gwtheta"], g["gwphi"], g["mc"], dist, g["fgw"], g["phase0"], g["psi"], g["inc"],
                             pdist=pdist, pphase=pph, evolve=False)
            src = CO.source_scalars(g["fgw"], g["mc"], g["h0"], g["phase0"], g["psi"], g["inc"])
            np.testing.assert_allclose(src, a["src"][:10], rtol=1e-13, atol=0)
            # the derived distance makes cgw_inputs' fac3 the drawn h0: fac3 = h0 / (2 w0^(2/3))
            np.testing.assert_allclose(a["src"][3] * 2 * a["src"][0] ** (2 / 3), g["h0"], rtol=1e-13)
            par = CO.pulsar_constants(phat, g["gwtheta"], g["gwphi"], g["fgw"], pdist, pph)
            np.testing.assert_allclose(par[:, 2], a["par"][:, 2], rtol=0, atol=1e-15)
            np.testing.assert_allclose(par[:, [0, 1]], a["par"][:, [0, 1]], rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(par[:, 3], a["par"][:, 3], rtol=1e-12)


def test_pole_gives_zero_pattern():
    from pta_replicator_b200 import orf
    b = _batch()
    locs = orf.psrlocs_from_pulsars(b.psrs)
    th, ph = np.pi / 2 - locs[:, 1], locs[:, 0]
    phat = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], axis=1)
    # a source in pulsar 1's direction (gwtheta, gwphi = the pulsar's: 1 + Omega.p = 0) and one antipodal to it (0/0)
    for gt, gp in ((th[1], ph[1]), (np.pi - th[1], (ph[1] + np.pi) % (2 * np.pi))):
        par = CO.pulsar_constants(phat, gt, gp, 1e-8, 1.0, pphase=np.full(3, 1.0))
        assert np.all(np.isfinite(par))
        assert par[1, 0] == 0.0 and par[1, 1] == 0.0 and par[1, 3] == 0.0


# ------------------------------------------------------------------ registration
def test_registration_and_removal():
    b = _batch()
    assert b._cwpop is None
    b._compiled = "x"
    b.set_cw_population(n_sources=2, pdist=[1.0, 2.0, 3.0], pphase="uniform", evolve=True)
    assert b._compiled is None
    cp = b._cwpop
    assert cp["n_src"] == 2 and cp["pphase"] and cp["mode"] == 0 and cp["psr_term"] == 1
    assert cp["kind"] == [CO.UNIFORM, CO.UNIFORM, CO.FIXED, CO.ACOS, CO.UNIFORM, CO.UNIFORM, CO.UNIFORM, CO.ACOS]
    assert cp["lo"][0] == -15.0 and cp["width"][0] == 2.0 and cp["lo"][2] == 9.0
    b.set_cw_population(phase_approx=True, psrTerm=False)
    assert b._cwpop["mode"] == 1 and b._cwpop["psr_term"] == 0
    b.set_cw_population()
    assert b._cwpop["mode"] == 2
    b._compiled = "x"
    b.set_cw_population(None)
    assert b._cwpop is None and b._compiled is None


@pytest.mark.parametrize("kw", [
    dict(log10_h0=(-13.0, -15.0)), dict(log10_fgw=(-8.0, -8.0)), dict(log10_mc=(9.0,)), dict(log10_mc=(1, 2, 3)),
    dict(log10_h0=float("nan")), dict(log10_fgw=(-9.0, float("inf"))), dict(log10_mc=None), dict(log10_h0="x"),
    dict(log10_h0=400.0),
    dict(gwtheta=-0.1), dict(gwtheta=(0.0, 3.2)), dict(gwphi=6.3), dict(phase0=(-1.0, 1.0)), dict(psi=3.2),
    dict(inc=(0.0, 4.0)), dict(gwtheta=float("nan")),
    dict(n_sources=0), dict(n_sources=65), dict(n_sources=1.5), dict(n_sources=True),
    dict(pdist=[1.0, 2.0]), dict(pdist=np.ones((3, 1))), dict(pdist=-1.0), dict(pdist=float("nan")),
    dict(pphase="random"), dict(pphase=1.0), dict(tref=float("inf")),
])
def test_bad_arguments_raise(kw):
    b = _batch()
    with pytest.raises(ValueError):
        b.set_cw_population(**kw)
    assert b._cwpop is None


def test_plan_only_device_calls_raise():
    from pta_replicator_b200 import _cabi
    b = _batch()
    b.set_cw_population(n_sources=4)
    b.plan()
    with pytest.raises(_cabi.PtarError):
        b.cw_population_params(8)
    with pytest.raises(_cabi.PtarError):
        b.generate(8)
