"""Chromatic noise in the generator on the H100: parity mode and every throughput build (WHITE x DET, rc 16 and 32,
fused and two-kernel, on the device's own PTAR_K_CHROM draws) at edge shapes against the extended-precision reference of
tests/generator_reference.py (each slot is a red-noise-like quadratic scaled by its per-TOA weight), the schedules bit for
bit, generate_to_host, every other draw unchanged by adding chromatic noise, the drop-ins against the numpy formula
w ⊙ F s z, the Taylor error at ng15 cadence, the chromatic spectrum at full size, and the optimal statistic and the
red-noise likelihood calibrated with a loud DM process injected and modelled."""
import numpy as np
import pytest

from tests import generator_reference as GR
from tests.test_chromatic_cpu import chrom_pulsars

pytestmark = pytest.mark.gpu

REPORT = GR.Report()


def _np(t):
    return t.detach().cpu().numpy()


def _batch(ntoas, red=6, dm=(), ch=(), white=True, ecorr=True, equad=None, det=False, **kw):
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(chrom_pulsars(ntoas, seed=3), **kw)
    T = float(np.ptp(np.concatenate(b.t_tdb)))
    with np.errstate(divide="ignore", invalid="ignore"):   # a 1-TOA pulsar's own span is 0 (fixed below)
        for i in range(b.n_psr):
            if white:
                b.set_white(i, efac=1.1, log10_equad=equad)
            if ecorr:
                b.set_ecorr(i, -6.4, coarsegrain=1.0 / 86400.0)
            if red:
                b.set_red(i, -13.9, 3.7, modes=np.arange(1, red + 1) / T)
            if i in dm:
                b.set_dm_noise(i, -13.3, 2.4, modes=np.arange(1, 9) / T)
            if i in ch:
                b.set_chromatic_noise(i, -13.6, 3.2, idx=4.0, modes=np.arange(1, 6) / T)
            if det:
                t = b.t_tdb[i]
                b.set_deterministic(i, (1e-7 * np.sin(2 * np.pi * (t - t[0]) / 3e7))[np.argsort(b.order[i])])
    # a 1-TOA pulsar has no span of its own, so its prior 1/T is infinite: it takes the longest pulsar's
    longest = int(np.argmax(b.ntoa))
    for c in [b._red] + b._chrom:
        if c is not None and c["f"][longest] is not None:
            c["scale"] = [c["scale"][longest] if s is not None and not np.all(np.isfinite(s)) else s for s in c["scale"]]
    return b


# a 1-TOA pulsar, a pulsar without chromatic noise next to one with both slots, > 1024 TOAs and > 64 epochs per pulsar
NTOAS = (1, 7, 40, 1100, 300)
DM, CH = (0, 2, 3, 4), (2, 3)


def _reference(b, st, D, R, merged=False):
    """check dict of the full output: the achromatic recipe plus sum_s w_s * (slot s as a red-noise process)."""
    from tests.test_gpu_generator_edges import _statics
    S = _statics(b, st, merged=merged, G=None)
    base, written = GR.generate(S, D, R)
    h, lo, bnd, mag = base["hi"].copy(), base["lo"].copy(), base["bound"].copy(), base["terms"].copy()
    zoff = 0
    for s, d in enumerate(st["chrom"]["slots"]):
        J = d["J"]
        Ss = dict(S, flags=GR.F_RED, J=J, conv=0, Ftile=_np(d["Ftile"]), rn_scale=_np(d["scale"]).reshape(b.n_psr, J),
                  rn_omega=_np(d["omega"]).reshape(b.n_psr, J // 2))
        q, _ = GR.generate(Ss, dict(zrn=D["zchr"][:, :, zoff:zoff + J]), R)
        w = _np(d["weight"])[None, :]
        ph, pl = GR.two_prod(q["hi"], np.broadcast_to(w, q["hi"].shape))
        h, lo = GR.pair_add(h, lo, ph, pl + w * q["lo"])
        bnd = bnd + np.abs(w) * q["bound"]
        mag = mag + np.abs(w) * q["terms"]
        zoff += J
    return dict(hi=h, lo=lo, bound=bnd + GR.gamma(8) * mag, terms=mag), written


def _inject(b, st, R, seed):
    import torch
    rng = np.random.default_rng(seed)
    Jc = sum(st["chrom"]["J"])
    D = dict(z1=rng.standard_normal((R, b.ld)), z2=rng.standard_normal((R, b.ld)),
             zb=rng.standard_normal((R, max(st["n_bucket_total"], 1))),
             zrn=rng.standard_normal((R, b.n_psr, max(st["J"], 2))), zchr=rng.standard_normal((R, b.n_psr, Jc)))
    return D, {k: torch.from_numpy(v) for k, v in D.items()}


@pytest.mark.parametrize("R", [5, 33])
def test_parity_against_reference_and_schedules_agree(R):
    import torch
    b = _batch(NTOAS, dm=DM, ch=CH)
    st = b.compile()
    D, inj = _inject(b, st, R, seed=11)
    outs = {}
    for sched, rc, split in (("fused", 0, False), ("rc32", 32, False), ("two_kernel", 0, True), ("two_kernel32", 32, True)):
        b.split_epoch = split
        outs[sched] = b.generate(R, inject=inj, rc=rc)
    b.split_epoch = False
    ref, written = _reference(b, st, D, R)
    got = _np(outs["fused"])
    GR.check(got[:, written], {k: v[:, written] for k, v in ref.items()}, f"chromatic parity R={R}", REPORT, "gen_chrom")
    for k in ("rc32", "two_kernel", "two_kernel32"):   # parity mode runs the rc = 16 builds: every schedule bit for bit
        assert torch.equal(outs[k], outs["fused"]), k


def test_throughput_schedules_agree_and_rc32():
    import torch
    b = _batch(NTOAS, dm=DM, ch=CH)
    ref = b.generate(64, seed=5)
    b.split_epoch = True
    assert torch.equal(b.generate(64, seed=5), ref)
    b.split_epoch = False
    r32 = b.generate(64, seed=5, rc=32)
    b.split_epoch = True
    assert torch.equal(b.generate(64, seed=5, rc=32), r32)
    assert torch.isfinite(ref).all()


def test_other_draws_unchanged():
    """generate(recipe + chromatic) - generate(recipe) == generate(chromatic only), same seed, to fp64 rounding (the
    chromatic window moves epoch references, so the red noise's Taylor step changes at its 1e-13 rms tolerance)."""
    full = _batch(NTOAS, dm=DM, ch=CH)
    base = _batch(NTOAS)
    only = _batch(NTOAS, red=0, dm=DM, ch=CH, white=False, ecorr=False)
    R = 48
    a, c, o = (_np(x.generate(R, seed=9)) for x in (full, base, only))
    scale = np.abs(a).max()
    d = np.abs((a - c) - o)
    assert d.max() <= 1e-11 * scale, d.max() / scale
    assert np.abs(o).max() > 1e-3 * scale   # the chromatic term is there


def test_dropins_match_the_numpy_formula():
    from pta_replicator_b200 import red_noise
    from pta_replicator_b200.engine import _sincos_basis
    for fn, idx, kw in ((red_noise.add_dm_noise, 2.0, {}), (red_noise.add_chromatic_noise, 4.4, dict(idx=4.4))):
        p = chrom_pulsars((120,), seed=8)[0]
        t = np.asarray(p.toas.table["tdbld"], np.float64) * 86400.0
        nu = np.asarray(p.toas.freq, dtype=float)
        fn(p, -13.0, 3.0, components=7, seed=42, fref=1300.0, **kw)
        np.random.seed(42)
        z = np.random.randn(14)
        T = t.max() - t.min()
        f = np.arange(1, 8) / T
        ff = np.repeat(f, 2)
        from pta_replicator_b200 import constants as const
        prior = 10 ** -26.0 * (ff / (1 / const.YEAR_IN_SEC)) ** -3.0 / (12 * np.pi ** 2 * T) * const.YEAR_IN_SEC ** 3
        want = (1300.0 / nu) ** idx * (_sincos_basis(t, f) @ (np.sqrt(prior) * z))
        got = p.toas.delay_s
        assert np.allclose(got, want, rtol=0, atol=1e-10 * np.abs(want).max()), fn.__name__
        assert any(k.endswith("_gp") for k in p.added_signals), p.added_signals.keys()


def test_taylor_error_against_exact_epochs():
    """Default epochs against exact_epochs=True on the same draws: within 1e-12 of the output scale."""
    a = _batch(NTOAS, dm=DM, ch=CH)
    e = _batch(NTOAS, dm=DM, ch=CH, exact_epochs=True)
    st_a, st_e = a.compile(), e.compile()
    R = 8
    D, inj = _inject(a, st_a, R, seed=2)
    ga, ge = _np(a.generate(R, inject=inj)), _np(e.generate(R, inject=inj))
    assert np.abs(ga - ge).max() <= 1e-12 * np.abs(ge).max()
    assert st_e["n_epochs"] > st_a["n_epochs"]


def test_shared_memory_refusal_is_a_value_error():
    b = _batch((30, 20), red=60, dm=(0,), ch=(0,))   # red noise alone fits rc = 32; with the chromatic block it does not
    with pytest.raises(ValueError, match="chromatic bases"):
        b.generate(32, seed=1, rc=32)


# ------------------------------------------------------------------ throughput builds on the device's own draws
def _chrom_draws(b, st, R, real0, seed):
    """zchr [R, P, sum J_s] of the device's stream: ptar_philox_normals(PTAR_K_CHROM, psr, realization, idx0 = s << 16)."""
    import torch
    from pta_replicator_b200 import _cabi
    L = _cabi.lib()
    cols = []
    for s, J in enumerate(st["chrom"]["J"]):
        z = np.zeros((R, b.n_psr, J))
        out = torch.empty(J, dtype=torch.float32, device=b.device)
        for p in range(b.n_psr):
            for r in range(R):
                _cabi.check(L.ptar_philox_normals(out.data_ptr(), _cabi.K_CHROM, p, real0 + r, s << 16, J, seed,
                                                  _cabi.current_stream()))
                z[r, p] = _np(out).astype(np.float64)
        cols.append(z)
    return np.concatenate(cols, axis=2)


BUILDS = [("w0d0", dict(white=False)), ("w0d1", dict(white=False, det=True)), ("w1d0", dict()), ("w1d1", dict(det=True)),
          ("w2d0", dict(equad=-6.5)), ("w2d1", dict(equad=-6.5, det=True))]


@pytest.mark.parametrize("sched", ["fused", "two_kernel"])
@pytest.mark.parametrize("rc", [16, 32])
@pytest.mark.parametrize("key,kw", BUILDS)
def test_throughput_builds_against_reference(key, kw, rc, sched):
    """Every throughput build (WHITE 0 / 1 / 2 x DET 0 / 1) at rc 16 and 32, fused and two-kernel, on the device's own
    draws -- white, ECORR and red noise from their streams, the slots from PTAR_K_CHROM -- against the reference."""
    from tests.test_gpu_generator_edges import _philox_draws
    b = _batch(NTOAS, dm=DM, ch=CH, **kw)
    two = key.startswith("w2")
    b.white_merged = not two
    b.split_epoch = sched == "two_kernel"
    st = b.compile()
    R, real0, seed = 37, 8, 13
    got = _np(b.generate(R, seed=seed, real0=real0, rc=rc))
    D = _philox_draws(b, st, R, real0, seed, two=two)
    D["zchr"] = _chrom_draws(b, st, R, real0, seed)
    ref, written = _reference(b, st, D, R, merged=not two)
    GR.check(got[:, written], {k: v[:, written] for k, v in ref.items()}, f"chromatic {key} rc={rc} {sched}", REPORT,
             f"gen_chrom_{sched}_rc{rc}")


def test_slots_draw_distinct_streams():
    """The two slots and the red noise draw different normals for the same pulsar, column and realization."""
    from pta_replicator_b200 import _cabi
    b = _batch((40,), dm=(0,), ch=(0,))
    st = b.compile()
    z = _chrom_draws(b, st, 4, 0, 3)
    J0 = st["chrom"]["J"][0]
    n = min(J0, z.shape[2] - J0)
    assert not np.any(z[:, :, :n] == z[:, :, J0:J0 + n])
    from tests.test_gpu_generator_edges import _philox
    zr = _philox(b, _cabi.K_RED, 0, 4, 0, n, 3)
    assert not np.any(zr == z[:, 0, :n])


def test_generate_to_host_equals_generate():
    """ptar_run_job_to_host_chrom (chunks, the copy overlapped) gives generate's rows bit for bit, with and without a
    timing-model fit."""
    b = _batch(NTOAS, dm=DM, ch=CH)
    R = 40
    for tm in (False, True):
        if tm:
            for i in range(b.n_psr):
                if b.ntoa[i] > 3:
                    b.set_timing_model(i, poly=2)
        dev = _np(b.generate(R, seed=21))
        host = b.generate_to_host(R, seed=21, chunk=12).numpy()
        assert np.array_equal(dev, host), tm


# ------------------------------------------------------------------ full size
@pytest.fixture(scope="module")
def ng15_sub():
    """ng15-full with each epoch's sub-band TOAs spread over its backend's band."""
    from pta_replicator_b200 import synthetic
    psrs, noise = synthetic.make_ng15_like("full")
    synthetic.spread_subband_frequencies(psrs)
    return psrs, noise


def _ng15_batch(ng15_sub, dm=None, chrom=None, **kw):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = ng15_sub
    recipe = {k: kw.pop(k) for k in ("white", "ecorr", "red", "gwb") if k in kw}
    npsr = kw.pop("npsr", len(psrs))
    b = synthetic.ng15_recipe(PulsarBatch(psrs[:npsr], **kw), noise, **recipe)
    for i in range(b.n_psr):
        if dm is not None:
            b.set_dm_noise(i, *dm)
        if chrom is not None and i % 3 == 0:
            b.set_chromatic_noise(i, *chrom)
    return b


TAYLOR = 1e-11   # max |d| / rms(pulsar): Taylor epochs vs one epoch per TOA, same draws (test_gpu_statistics.py)


def test_fullsize_taylor_epochs_against_exact_epochs(ng15_sub):
    """Red noise + DM on every pulsar + scattering on every third, no white noise and no ECORR (so the processes'
    windows alone decide the epochs): default epochs against exact_epochs=True on the same Philox draws,
    max |d| / rms(pulsar) < TAYLOR."""
    kw = dict(white=False, ecorr=False, gwb=False, dm=(-13.0, 2.0), chrom=(-13.5, 2.5, 4.0))
    ref_b = _ng15_batch(ng15_sub, exact_epochs=True, **kw)
    ref = ref_b.generate(16, seed=99, real0=32)
    del ref_b
    b = _ng15_batch(ng15_sub, **kw)
    n_toa, n_ep = b.n_toa_total, b.compile()["n_epochs"]
    assert n_ep < n_toa   # sub-band TOAs share epochs
    got = b.generate(16, seed=99, real0=32)
    worst = 0.0
    for i in range(b.n_psr):
        sl = slice(b.toa_off[i], b.toa_off[i] + b.ntoa[i])
        worst = max(worst, ((got[:, sl] - ref[:, sl]).abs().max() / ref[:, sl].std()).item())
    print(f"\n[chrom] Taylor epochs ({n_ep} for {n_toa} TOAs) vs exact epochs: max|d|/rms = {worst:.3e}")
    assert worst < TAYLOR, worst


def test_fullsize_chromatic_spectrum(ng15_sub):
    """DM only, 2048 realizations: the least-squares coefficients of the residuals on the weighted basis w ⊙ F of every
    tenth pulsar have per-frequency power sum_r (a_sin^2 + a_cos^2) / prior ~ chi^2_{2R} within 5 sigma, and the
    log-log slope of the power equals -gamma within 0.05 (as test_fullsize_red_noise_spectrum for red noise)."""
    import torch
    from pta_replicator_b200 import constants as const
    log10_A, gamma = -13.2, 2.5
    b = _ng15_batch(ng15_sub, white=False, ecorr=False, red=False, gwb=False, dm=(log10_A, gamma, 30))
    R = 2048
    x = b.generate(R, seed=17)
    for i in range(0, b.n_psr, 10):
        s, n = b.toa_off[i], b.ntoa[i]
        t = torch.from_numpy(b.t_tdb[i]).to(x.device)
        T = float(b.t_tdb[i].max() - b.t_tdb[i].min())
        f = torch.arange(1, 31, dtype=torch.float64, device=x.device) / T
        arg = 2 * np.pi * t[:, None] * f[None, :]
        w = torch.from_numpy((1400.0 / b.freq[i]) ** 2).to(x.device)[:, None]
        F = torch.empty((n, 60), dtype=torch.float64, device=x.device)
        F[:, 0::2], F[:, 1::2] = w * torch.sin(arg), w * torch.cos(arg)
        y = x[:, s:s + n].T.contiguous()
        a = torch.linalg.lstsq(F, y).solution
        resid = (F @ a - y).abs().max().item() / y.std().item()
        assert resid < 1e-9, resid
        fk = f.cpu().numpy()
        prior = 10 ** (2 * log10_A) * (fk * const.YEAR_IN_SEC) ** (-gamma) * const.YEAR_IN_SEC ** 3 / (12 * np.pi ** 2 * T)
        power = (a[0::2] ** 2 + a[1::2] ** 2).sum(1).cpu().numpy()
        chi = power / prior
        assert np.all(np.abs(chi / (2 * R) - 1) < 5 / np.sqrt(R)), (i, chi / (2 * R))
        slope = np.polyfit(np.log(fk), np.log(power), 1)[0]
        assert abs(slope + gamma) < 0.05, (i, slope)


def test_optimal_statistic_calibrated_with_dm_noise_modelled(ng15_sub):
    """White + ECORR + red noise + a loud DM process on every pulsar (modelled), timing models, no GWB: the noise-only
    S/N of every template over 4096 realizations has mean 0 and variance 1 within 4 sigma."""
    b = _ng15_batch(ng15_sub, gwb=False, dm=(-12.5, 2.5, 30))
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    b.set_optimal_statistic()
    R = 4096
    snr = b.optimal_statistic(R, seed=20250923)["snr"].cpu().numpy()
    mean, var = snr.mean(axis=0), snr.var(axis=0, ddof=1)
    print(f"\n[chrom] OS null with loud DM modelled, R={R}: S/N mean {np.round(mean, 4)}, var {np.round(var, 4)}")
    assert np.all(np.abs(mean) < 4 / np.sqrt(R))
    assert np.all(np.abs(var - 1) < 4 * np.sqrt(2.0 / (R - 1)))


def test_red_noise_likelihood_law_with_dm_only(ng15_sub):
    """Pulsars carrying white + ECORR + a loud DM process and no red noise: the red-noise likelihood models the DM
    process as noise, so Q = 2 lnL + ldet follows its noise-only law exactly (test_null_law_of_q's check), and the
    ln B against noise stays in that law's range."""
    from tests.test_gpu_red_noise_likelihood import _law
    b = _ng15_batch(ng15_sub, npsr=4, red=False, gwb=False, dm=(-12.5, 2.5, 30))
    x, gam = np.array([-15.0, -14.0, -13.0]), np.array([2.0, 13 / 3, 6.0])
    b.set_red_noise_likelihood(log10_A=x, gamma=gam)
    pr = b.plan()["rn"]
    res = b.red_noise_likelihood(4096, seed=20250924, maps=True)
    Qs = 2 * res["lnL"].cpu().numpy() + pr["ldet"][None]
    _law(b, pr, Qs, pr["Z"], "H0 with DM", range(3), range(3))
