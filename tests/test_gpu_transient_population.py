"""Per-realization burst-with-memory and sine-Gaussian burst populations on the device (``set_bwm_population``,
``set_burst_population``, ``ptar_transient_population``): the draws against the numpy restatement of tests/tpop_oracle.py,
the injection against an extended-precision evaluation of the add kernel's formula on edge shapes (noise before t0 and
alignment slots untouched, finite rows at a pulsar's pole), chunk / real0 / path invariance, the timing fit, the
searches' conventions on noise-free rows, the noncentral law of B under the population, removal and refusals."""
import ctypes as C

import numpy as np
import pytest

from tests import deterministic_reference as DR
from tests import tpop_oracle as TO
from tests.reduction_reference import U, gamma
from tests.test_gpu_burst_statistic import _pulsars
from tests.test_gpu_cw_population import _cgw_batch, _np, _slots

pytestmark = pytest.mark.gpu

SEED = 20261019
K_EXP = 1   # CUDA's documented maximum ulp error of double exp


def _set(b, family, **kw):
    (b.set_bwm_population if family == "bwm" else b.set_burst_population)(**kw)


def _params(b, family, R, seed=SEED, real0=0):
    p = (b.bwm_population_params if family == "bwm" else b.burst_population_params)(R, seed=seed, real0=real0)
    return {k: _np(v) for k, v in p.items()}


def _pop(b, family):
    return b._bwmpop if family == "bwm" else b._burstpop


# ------------------------------------------------------------------ draws
@pytest.mark.parametrize("family", ("bwm", "burst"))
def test_params_equal_numpy_restatement(family):
    b = _cgw_batch(3)
    _set(b, family, n_sources=5, gwtheta=(0.2, 2.9) if family == "bwm" else None)
    R, r0 = 300, 1001
    got = _params(b, family, R, real0=r0)
    ref = TO.draw(_pop(b, family), np.arange(r0, r0 + R), SEED)
    if family == "bwm":
        exact = dict(t0_mjd=TO.T0, log10_strain=TO.LOG10_AMP, gwtheta=TO.GWTHETA, gwphi=TO.GWPHI, bwm_pol=TO.POL)
    else:
        exact = dict(t0_mjd=TO.T0, log10_amp=TO.LOG10_AMP, log10_f0=TO.LOG10_F0, Q=TO.Q, gwphi=TO.GWPHI, psi=TO.POL,
                     phase0=TO.PHASE0, eps=TO.EPS)
        g = ref[..., TO.GWTHETA]
        assert np.all(np.abs(got["gwtheta"] - g) <= 4 * np.spacing(np.abs(g)))     # through acos
        f0 = 10.0 ** ref[..., TO.LOG10_F0]
        np.testing.assert_allclose(got["f0"], f0, rtol=1e-15)
        np.testing.assert_allclose(got["tau"], ref[..., TO.Q] / (2 * np.pi * f0), rtol=1e-14)
        a = np.stack([TO.search_amplitudes(v) for v in ref.reshape(-1, TO.NPAR)]).reshape(R, 5, 4)
        A = 10.0 ** ref[..., TO.LOG10_AMP]
        assert np.all(np.abs(got["a"] - a) <= 1e-14 * A[..., None])
    for k, j in exact.items():
        assert np.array_equal(got[k], ref[..., j]), k                                # affine maps: bit for bit
    amp = "strain" if family == "bwm" else "amp"
    np.testing.assert_allclose(got[amp], 10.0 ** ref[..., TO.LOG10_AMP], rtol=1e-15)


# ------------------------------------------------------------------ injection against the extended-precision reference
def _exp(x):
    v = np.exp(x.v)
    return DR.E(v, np.abs(v).astype(np.float64) * x.e + K_EXP * 2 * U * np.abs(v).astype(np.float64))


def _operands(b, family, R):
    """The add kernel's operands as the draw left them in the population's scratch (one chunk of R realizations):
    rec [R, S, 4], coef [R, S, P, 2]."""
    key = family + "pop"
    S, P = _pop(b, family)["n_src"], b.n_psr
    scr = _np(b._scratch(key, 0))
    return scr[:R * S * 4].reshape(R, S, 4), scr[R * S * 4:R * S * (4 + 2 * P)].reshape(R, S, P, 2)


def _check_coefficients(b, family, coef, prm_ref):
    """coef against the restated coefficients of the device's own parameters."""
    phat = b._phat()
    for r in range(coef.shape[0]):
        for s in range(coef.shape[1]):
            c = TO.coefficients(TO.BWM if family == "bwm" else TO.BURST, prm_ref[r, s], phat)
            A = 10.0 ** prm_ref[r, s, TO.LOG10_AMP]
            np.testing.assert_allclose(coef[r, s], c, rtol=0, atol=1e-12 * A)


def _reference(family, rec, coef, t, pid, r):
    """sum_s term(r, s, t) as the add kernel evaluates it, in E arithmetic over the slots (t, pid); returns (value,
    bound, sum |term|, mask of the slots with at least one evaluated term)."""
    S = rec.shape[1]
    v = np.zeros(len(t), dtype=np.longdouble)
    e, a_sum, hit = np.zeros(len(t)), np.zeros(len(t)), np.zeros(len(t), dtype=bool)
    for s in range(S):
        q, c = rec[r, s], coef[r, s][pid]
        if family == "bwm":
            on = ~(t < q[0])
            term = DR.E(c[:, 0]) * (DR.E(t) - DR.E(q[0]))
        else:
            dt = DR.E(t) - DR.E(q[0])
            x = dt * DR.E(q[2])
            ee = x * x
            on = (t - q[0]) * q[2] * ((t - q[0]) * q[2]) < 750.0
            arg = dt * DR.E(q[1]) + DR.E(q[3])
            term = _exp(-ee) * (DR.E(c[:, 0]) * DR.EK.cos(arg) + DR.E(c[:, 1]) * DR.EK.sin(arg))
        v += np.where(on, term.v, 0)
        e += np.where(on, term.e, 0)
        a_sum += np.where(on, np.abs(term.v), 0).astype(np.float64)
        hit |= on
    return v, e, a_sum, hit


def _check_injection(b, family, with_, without, R, what):
    sel, pad = _slots(b)
    assert np.array_equal(with_[:, pad], without[:, pad]), what                 # alignment slots untouched
    t = np.concatenate([m * 86400 for m in b.mjd])
    pid = np.concatenate([np.full(n, i) for i, n in enumerate(b.ntoa)])
    rec, coef = _operands(b, family, R)
    ref = TO.draw(_pop(b, family), np.arange(R), SEED)
    _check_coefficients(b, family, coef, ref)
    assert np.array_equal(rec[..., 0], ref[..., TO.T0] * 86400.0)
    worst = 0.0
    for r in range(R):
        v, e, a_sum, hit = _reference(family, rec, coef, t, pid, r)
        w, wo = with_[r, sel], without[r, sel]
        assert np.array_equal(w[~hit], wo[~hit]), f"{what} r={r}: a slot without a term changed"
        d = w - wo
        bound = e + gamma(rec.shape[1] + 1) * a_sum + 2 * U * (np.abs(w) + np.abs(d))
        err = np.abs((d - v).astype(np.float64))
        ratio = np.where(err == 0, 0.0, err / bound)
        k = int(np.argmax(ratio))
        assert ratio[k] <= 1.0, f"{what} r={r}: |d|/bound {ratio[k]:.3g} at slot {sel[k]}: {d[k]!r} vs {v[k]!r}"
        worst = max(worst, float(ratio.max()))
    return worst


@pytest.mark.parametrize("P", (1, 3))
@pytest.mark.parametrize("family", ("bwm", "burst"))
def test_injection_against_reference(family, P):
    b = _cgw_batch(P)
    R = 6
    without = _np(b.generate(R, seed=SEED))
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    amp = dict(log10_strain=(-14.0, -12.0)) if family == "bwm" else dict(log10_amp=(-7.0, -6.0))
    worst = 0.0
    for S in (1, 3):
        for narrow in (False, True):
            kw = dict(amp)
            if family == "burst" and narrow:   # short bursts: g underflows on most of the span, terms are skipped
                kw.update(log10_f0=float(np.log10(200 / ((last - first) * 86400))), Q=(0.5, 1.0))
            if family == "bwm" and narrow:     # epochs late in the span: most slots lie before every t0
                kw.update(t0_mjd=(first + 0.8 * (last - first), last))
            _set(b, family, n_sources=S, **kw)
            rows = _np(b.generate(R, seed=SEED))
            assert np.isfinite(rows).all()
            worst = max(worst, _check_injection(b, family, rows, without, R, f"{family} P={P} S={S} narrow={narrow}"))
    print(f"\n[tpop] {family} P={P}: worst |d|/bound {worst:.3f}")
    _set(b, family, n_sources=None)
    assert np.array_equal(_np(b.generate(R, seed=SEED)), without)


@pytest.mark.parametrize("family", ("bwm", "burst"))
def test_source_at_a_pulsar_pole_is_finite(family):
    from pta_replicator_b200 import orf
    b = _cgw_batch(3)
    loc = orf.psrlocs_from_pulsars(b.psrs)[1]
    without = _np(b.generate(8, seed=SEED))
    first = min(m.min() for m in b.mjd)
    for gt, gp in ((np.pi / 2 - loc[1], loc[0]), (np.pi / 2 + loc[1], (loc[0] + np.pi) % (2 * np.pi))):
        _set(b, family, n_sources=2, gwtheta=gt, gwphi=gp, t0_mjd=first + 1.0)
        rows = _np(b.generate(8, seed=SEED))
        assert np.isfinite(rows).all()
        s = slice(b.toa_off[1], b.toa_off[1] + b.ntoa[1])
        assert np.array_equal(rows[:, s], without[:, s])                      # pattern (0, 0) at that pulsar
        assert not np.array_equal(rows, without)


# ------------------------------------------------------------------ invariance, paths and the timing fit
def _search_batch(P=6, tm=False, nep=40):
    from tests.test_gpu_burst_statistic import _batch
    return _batch(_pulsars(P, nep=nep), tm=tm, red=False)


def test_chunk_real0_and_path_invariance():
    import torch
    b = _search_batch()
    b.set_bwm_statistic(n_epochs=16, nside=2)
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    mid = 0.5 * (first + last)
    b.set_burst_statistic(t0_mjd=[mid, mid + 100.0], f0=[6.0 / ((last - first) * 86400)] * 2, Q=[5.0, 5.0], nside=2)
    b.set_bwm_population(n_sources=3)
    b.set_burst_population(n_sources=2)
    full = b.generate(32, seed=SEED, chunk=8)
    part = b.generate(16, seed=SEED, real0=8)
    assert torch.equal(full[8:24], part)
    for fn in (b.bwm_population_params, b.burst_population_params):
        pf, pp = fn(32, seed=SEED), fn(16, seed=SEED, real0=8)
        for k in pf:
            assert torch.equal(pf[k][8:24], pp[k]), k
    for stat, of in ((b.bwm_statistic, b.bwm_statistic_of), (b.burst_statistic, b.burst_statistic_of)):
        a = stat(16, seed=SEED, real0=8, chunk=12)
        c = of(part)
        for k, v in a.items():
            if isinstance(v, torch.Tensor):
                assert torch.equal(v, c[k]), k
    # each population alone is what it adds on top of the other
    b.set_burst_population(None)
    only_bwm = b.generate(16, seed=SEED, real0=8)
    b.set_bwm_population(None)
    plain = b.generate(16, seed=SEED, real0=8)
    assert not torch.equal(only_bwm, plain) and not torch.equal(part, only_bwm)


@pytest.mark.parametrize("family", ("bwm", "burst"))
def test_timing_fit_projects_the_injection(family):
    import torch
    from pta_replicator_b200 import _cabi
    b = _cgw_batch(3, ntoas=(65, 193, 1025))
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    R = 8
    post0 = b.generate(R, seed=SEED)
    pre0 = b._generate(R, SEED, 0, None, None, None, 0, None, postfit=False).clone()
    _set(b, family, n_sources=3)
    post1 = b.generate(R, seed=SEED)
    pre1 = b._generate(R, SEED, 0, None, None, None, 0, None, postfit=False).clone()
    inj = (pre1 - pre0).contiguous()
    scale = float(inj.abs().max())
    assert scale > 0
    tm = b.compile()["tm"]
    scratch = torch.empty(tm["n_tiles"] * R * tm["kmax"], dtype=torch.float64, device=b.device)
    _cabi.check(_cabi.lib().ptar_timing_project(inj.data_ptr(), b.ld, R, C.addressof(tm["model"]), scratch.data_ptr(),
                                                scratch.numel(), _cabi.current_stream()), "ptar_timing_project")
    err = float(((post1 - post0) - inj).abs().max())
    print(f"\n[tpop] {family} timing fit: max |(post-fit with - without) - fit(injection)| = {err:.3e} of {scale:.3e}")
    assert err <= 1e-12 * scale


# ------------------------------------------------------------------ the searches on the injected populations
def _cell_batch(family):
    """A 6-pulsar batch with its search registered, and a grid cell: (batch, cell dict, population kwargs)."""
    from pta_replicator_b200.engine import healpix_ring_centres
    b = _search_batch()
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    sky = healpix_ring_centres(2)
    s_star = 17
    if family == "bwm":
        b.set_bwm_statistic(n_epochs=24, nside=2)
        t0 = b._bwm["t0_mjd"]
        j_star = 9
        pop = dict(t0_mjd=float(t0[j_star]), gwtheta=sky[s_star, 0], gwphi=sky[s_star, 1])
    else:
        Tspan = (last - first) * 86400
        mid = 0.5 * (first + last)
        f0 = np.array([5.0, 5.0, 8.0, 8.0]) / Tspan
        t0 = np.array([mid, mid + 200.0, mid, mid - 150.0])
        b.set_burst_statistic(t0_mjd=t0, f0=f0, Q=[5.0, 5.0, 6.0, 6.0], nside=2)
        tm_ = b._burst["templates"]
        j_star = int(np.flatnonzero((tm_[:, 0] == mid) & (tm_[:, 1] == f0[2]))[0])
        pop = dict(t0_mjd=float(tm_[j_star, 0]), log10_f0=float(np.log10(tm_[j_star, 1])), Q=float(tm_[j_star, 2]),
                   gwtheta=sky[s_star, 0], gwphi=sky[s_star, 1])
    return b, dict(j=j_star, s=s_star), pop


def _noise_free(b, family, R, seed):
    """The rows the population adds in realizations [0, R) of ``seed`` (rows with it minus rows without)."""
    with_ = b.generate(R, seed=seed)
    saved = _pop(b, family)
    _set(b, family, n_sources=None)
    rows = with_ - b.generate(R, seed=seed)
    setattr(b, "_" + family + "pop", saved)
    b._compiled = None
    return rows


@pytest.mark.parametrize("family", ("bwm", "burst"))
def test_search_recovers_the_injected_parameters(family):
    """On noise-free rows of a source fixed on a search cell the argmax is that cell and the recovered amplitudes are
    the injected ones: a sign or polarisation-convention error between the injection and the search fails here."""
    b, cell, pop = _cell_batch(family)
    amp = dict(log10_strain=(-13.5, -12.5)) if family == "bwm" else dict(log10_amp=(-6.5, -6.0))
    _set(b, family, n_sources=1, **amp, **pop)
    R = 64
    rows = _noise_free(b, family, R, SEED)
    prm = _params(b, family, R)
    if family == "bwm":
        res = {k: _np(v) for k, v in b.bwm_statistic_of(rows).items() if hasattr(v, "cpu")}
        assert np.all(res["bwm_argmax_t0"] == cell["j"]) and np.all(res["bwm_argmax_sky"] == cell["s"])
        np.testing.assert_allclose(res["bwm_strain"], prm["strain"][:, 0], rtol=1e-9)
        dpol = np.angle(np.exp(2j * (res["bwm_pol"] - prm["bwm_pol"][:, 0]))) / 2      # mod pi
        assert np.all(np.abs(dpol) <= 1e-9), float(np.abs(dpol).max())
    else:
        res = {k: _np(v) for k, v in b.burst_statistic_of(rows).items() if hasattr(v, "cpu")}
        assert np.all(res["argmax_template"] == cell["j"]) and np.all(res["argmax_sky"] == cell["s"])
        a = prm["a"][:, 0]
        err = np.abs(res["amp"] - a).max(axis=1) / np.abs(a).max(axis=1)
        assert np.all(err <= 1e-9), float(err.max())


@pytest.mark.parametrize("family", ("bwm", "burst"))
def test_noncentral_law_at_the_cell(family):
    """With noise, 2B at the source's cell is noncentral chi^2_k(lambda_r), lambda_r = 2B of realization r's noise-free
    rows (k = 2 for BWM, 4 for the burst): the pooled z of sum_r (2B - k - lambda_r) lies within |z| < 5."""
    b, cell, pop = _cell_batch(family)
    R, k = 4096, 2 if family == "bwm" else 4
    stat, of, name = ((b.bwm_statistic, b.bwm_statistic_of, "bwm") if family == "bwm"
                      else (b.burst_statistic, b.burst_statistic_of, "B"))
    amp, a0 = ("log10_strain", -14.0) if family == "bwm" else ("log10_amp", -7.0)

    def lam_of(n):
        return 2.0 * _np(of(_noise_free(b, family, n, SEED), maps=True)[name][:, cell["j"], cell["s"]])

    _set(b, family, n_sources=1, **{amp: a0}, **pop)
    c = a0 + 0.5 * np.log10(20.0 / float(lam_of(256).mean()))     # lambda scales as amplitude^2: mean lambda ~ 20
    _set(b, family, n_sources=1, **{amp: (c - 0.5, c + 0.5)}, **pop)
    lam = lam_of(R)
    x = 2.0 * _np(stat(R, seed=SEED, maps=True)[name][:, cell["j"], cell["s"]])
    z = np.sum(x - k - lam) / np.sqrt(np.sum(2.0 * (k + 2 * lam)))
    print(f"\n[tpop] {family}: R={R}, median lambda {np.median(lam):.2f}, mean(2B - k - lambda) "
          f"{np.mean(x - k - lam):.3f}, z = {z:.2f}")
    assert np.median(lam) > 1.0
    assert abs(z) < 5


# ------------------------------------------------------------------ removal and refusals
def test_removal_and_refusals():
    import torch
    fresh = _cgw_batch(3)
    ref = fresh.generate(8, seed=SEED)
    b = _cgw_batch(3)
    for family in ("bwm", "burst"):
        _set(b, family, n_sources=2)
        with_ = b.generate(8, seed=SEED)
        assert not torch.equal(with_, ref)
        with pytest.raises(ValueError):
            b.generate(8, inject=dict(z1=torch.zeros(8, b.ld), z2=torch.zeros(8, b.ld)))
        with pytest.raises(ValueError, match="generate"):
            b.generate_to_host(8, seed=SEED)
        _set(b, family, n_sources=None)
        assert torch.equal(b.generate(8, seed=SEED), ref)
        with pytest.raises(ValueError):
            _params(b, family, 8)
