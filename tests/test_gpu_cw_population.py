"""Per-realization continuous-wave populations on the device (``set_cw_population``, ``ptar_cw_population``): the draws
against the numpy restatement of tests/cwpop_oracle.py, chunk and shard invariance, the injection against the
extended-precision CW reference of tests/deterministic_reference.py on edge shapes (noise untouched, alignment slots
untouched, finite rows at a pulsar's pole), the timing fit, the Fe-statistic end to end, removal and refusals."""
import ctypes as C

import numpy as np
import pytest

from tests import cwpop_oracle as CO
from tests import deterministic_reference as DR
from tests import generator_reference as GR
from tests.reduction_reference import EDGE_NTOAS, U, gamma

pytestmark = pytest.mark.gpu

SEED = 20261018


def _np(t):
    return t.detach().cpu().numpy()


def _cgw_batch(P, ntoas=None, **kw):
    """The dense edge batches of test_gpu_deterministic_edges (odd TOA counts, epochs straddling tiles), or pulsars of
    ``ntoas`` TOAs, with white noise."""
    from pta_replicator_b200.engine import PulsarBatch
    pool = GR.GEN_NTOAS + EDGE_NTOAS
    ntoas = ntoas or {1: (1025,), 3: (1, (17, 2), 2100)}.get(P) or tuple(pool[j % len(pool)] for j in range(P))
    b = PulsarBatch(GR.dense_pulsars(ntoas, seed=P, name="W"), **kw)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.0, log10_equad=-6.5)
    return b


def _slots(b):
    sel = np.concatenate([np.arange(o, o + n) for o, n in zip(b.toa_off, b.ntoa)])
    pad = np.ones(b.ld, dtype=bool)
    pad[sel] = False
    return sel, pad


# ------------------------------------------------------------------ draws
@pytest.mark.parametrize("pphase", (None, "uniform"))
def test_params_equal_numpy_restatement(pphase):
    b = _cgw_batch(3)
    b.set_cw_population(n_sources=5, log10_mc=(8.0, 10.0), gwtheta=None, inc=(0.1, 3.0), pphase=pphase)
    R, r0 = 300, 1001
    got = {k: _np(v) for k, v in b.cw_population_params(R, seed=SEED, real0=r0).items()}
    ref = CO.draw(b._cwpop, np.arange(r0, r0 + R), SEED, b.n_psr)
    for k in ("gwphi", "phase0", "psi", "inc", "log10_h0", "log10_fgw", "log10_mc") + (("pphase",) if pphase else ()):
        assert np.array_equal(got[k], ref[k]), k                               # affine maps: bit for bit
    ulp = np.spacing(np.abs(ref["gwtheta"]))
    assert np.all(np.abs(got["gwtheta"] - ref["gwtheta"]) <= 4 * ulp)        # through acos
    for k in ("h0", "fgw", "mc"):
        np.testing.assert_allclose(got[k], ref[k], rtol=1e-15)
    np.testing.assert_allclose(got["dist"], CO.dist_mpc(got["h0"], got["fgw"], got["mc"]), rtol=1e-14)


# ------------------------------------------------------------------ chunk / shard invariance
def test_chunk_and_shard_invariance():
    import torch
    b = _cgw_batch(3, ntoas=(65, 193, 1025))     # every pulsar long enough for the Fp-statistic's statics
    b.set_fp_statistic(n_freqs=8)
    b.set_cw_population(n_sources=3, pphase="uniform", evolve=True)
    full = b.generate(32, seed=SEED, chunk=8)
    part = b.generate(16, seed=SEED, real0=8)
    assert torch.equal(full[8:24], part)
    pf = b.cw_population_params(32, seed=SEED)
    pp = b.cw_population_params(16, seed=SEED, real0=8)
    for k in pf:
        assert torch.equal(pf[k][8:24], pp[k]), k
    # the rows a statistic reduces, generated inside _rows_reduce at another chunk
    def outputs(st, R):
        return dict(rows=torch.empty((R, b.ld), dtype=torch.float64, device=b.device))

    def reduce(st, rows, n, res, r0, timers):
        res["rows"][r0:r0 + n].copy_(rows[:n])
    b._scratch("rows", 12 * b.ld).fill_(7.0)      # the statistics' shared row scratch, as an earlier call may leave it
    got = b._rows_reduce("fp", outputs, reduce, 16, SEED, 8, 12, None)["rows"]
    # the generator defines every slot up to the last pulsar's aligned end; the tail of the packed axis past it is left
    # as the caller's buffer had it (zeros from generate, the scratch's old contents in _rows_reduce), population or not
    used = b.toa_off[-1] + -(-b.ntoa[-1] // 4) * 4
    assert used < b.ld
    assert torch.equal(got[:, :used], part[:, :used])
    assert torch.all(part[:, used:] == 0) and torch.all(got[:, used:] == 7.0)
    b.set_cw_population(None)
    assert not torch.equal(b.generate(16, seed=SEED, real0=8), part)


# ------------------------------------------------------------------ injection against the extended-precision reference
def _source_inputs(b, prm, r, s, pdist, pphase):
    g = {k: float(prm[k][r, s]) for k in ("gwtheta", "gwphi", "phase0", "psi", "inc", "fgw", "mc", "dist")}
    pph = None if pphase is None else prm["pphase"][r, s]
    cp = b._cwpop
    return b.cgw_inputs(g["gwtheta"], g["gwphi"], g["mc"], g["dist"], g["fgw"], g["phase0"], g["psi"], g["inc"],
                        pdist=pdist, pphase=pph, psrTerm=bool(cp["psr_term"]), evolve=cp["mode"] == 0,
                        phase_approx=cp["mode"] == 1, tref=cp["tref"])


def _reference(b, a, sel):
    """cw_res on ``cgw_inputs`` of one drawn source, its operands carrying the error of the device's own derivation
    (a few ulp of each scalar; F+ and Fx from the other, pole-safe form of 1 + Omega.p).  Returns (value, bound) over
    the slots ``sel``; the monochromatic mode adds the error of its rotation by the pulsar-term phase offset."""
    src, par, pid = a["src"], a["par"], a["pid"][sel]
    q = [DR.E(src[k], 16 * U * abs(src[k])) for k in range(10)]
    den = np.abs(1 - par[:, 2])                        # |1 + Omega.p| = |1 - cosMu|
    ferr = 16 * U * (np.abs(par[:, :2]) + 1) / np.maximum(den, 1e-300)[:, None]
    q += [DR.E(par[pid, 0], ferr[pid, 0]), DR.E(par[pid, 1], ferr[pid, 1]), DR.E(par[pid, 2], 4 * U * np.ones(len(pid))),
          DR.E(par[pid, 3], 16 * U * np.abs(par[pid, 3]))]
    r = DR.cw_res(DR.EK, DR.E(a["t"][sel]), q, a["mode"], a["psr_term"])
    v, e = r.v, r.e
    if a["mode"] == 2 and a["psr_term"]:
        delta = 2 * src[0] * par[pid, 3] * (1 - par[pid, 2])
        amp = (np.abs(par[pid, 0]) + np.abs(par[pid, 1])) * abs(src[3] / np.cbrt(src[0])) * (abs(src[6]) + abs(src[7])) * 2
        e = e + amp * (8 * U * np.abs(delta) + 16 * U)
    return v, e


def _check_injection(b, rows_with, rows_without, prm, pdist, pphase, what):
    sel, pad = _slots(b)
    R, S = rows_with.shape[0], b._cwpop["n_src"]
    assert np.array_equal(rows_with[:, pad], rows_without[:, pad]), what     # alignment slots untouched
    diff = rows_with - rows_without
    worst = 0.0
    for r in range(R):
        v = np.zeros(len(sel), dtype=np.longdouble)
        e, a_sum = np.zeros(len(sel)), np.zeros(len(sel))
        for s in range(S):
            vs, es = _reference(b, _source_inputs(b, prm, r, s, pdist, pphase), sel)
            ok = ~np.isnan(vs)
            v += np.where(ok, vs, 0)
            e += np.where(ok, es, 0)
            a_sum += np.abs(np.where(ok, vs, 0)).astype(np.float64)
        bound = e + gamma(S + 1) * a_sum + 2 * U * (np.abs(rows_with[r, sel]) + np.abs(diff[r, sel]))
        d = np.abs((diff[r, sel] - v).astype(np.float64))
        ratio = np.where(d == 0, 0.0, d / bound)
        k = int(np.argmax(ratio))
        assert ratio[k] <= 1.0, f"{what} r={r}: |d|/bound {ratio[k]:.3g} at slot {sel[k]}: {diff[r, sel[k]]!r} vs {v[k]!r}"
        worst = max(worst, float(ratio.max()))
    return worst


@pytest.mark.parametrize("P", (1, 3))
def test_injection_against_reference(P):
    b = _cgw_batch(P)
    R = 6
    without = _np(b.generate(R, seed=SEED))
    pdist = np.linspace(0.5, 2.0, P)
    worst = {}
    for mode in (0, 1, 2):
        for psr_term in (False, True):
            for pphase in (None, "uniform"):
                for S in (1, 3):
                    b.set_cw_population(n_sources=S, log10_h0=(-14.5, -13.5), log10_fgw=(-8.7, -7.3), log10_mc=(8.5, 9.3),
                                        pdist=pdist, pphase=pphase, psrTerm=psr_term, evolve=mode == 0,
                                        phase_approx=mode == 1, tref=53000 * 86400.0 if S == 3 else 0)
                    rows = _np(b.generate(R, seed=SEED))
                    assert np.isfinite(rows).all()
                    prm = {k: _np(v) for k, v in b.cw_population_params(R, seed=SEED).items()}
                    w = _check_injection(b, rows, without, prm, pdist, pphase,
                                         f"P={P} mode={mode} psrTerm={psr_term} pphase={pphase} S={S}")
                    worst[mode] = max(worst.get(mode, 0.0), w)
    print(f"\n[cwpop] P={P}: worst |d|/bound per mode " + ", ".join(f"{m}: {w:.3f}" for m, w in sorted(worst.items())))
    b.set_cw_population(None)
    assert np.array_equal(_np(b.generate(R, seed=SEED)), without)


def test_source_at_a_pulsar_pole_is_finite():
    from pta_replicator_b200 import orf
    b = _cgw_batch(3)
    loc = orf.psrlocs_from_pulsars(b.psrs)[1]
    without = _np(b.generate(8, seed=SEED))
    for gt, gp in ((np.pi / 2 - loc[1], loc[0]), (np.pi / 2 + loc[1], (loc[0] + np.pi) % (2 * np.pi))):
        for mode in (0, 1, 2):
            b.set_cw_population(n_sources=2, gwtheta=gt, gwphi=gp, pphase="uniform", evolve=mode == 0,
                                phase_approx=mode == 1)
            rows = _np(b.generate(8, seed=SEED))
            assert np.isfinite(rows).all()
            s = slice(b.toa_off[1], b.toa_off[1] + b.ntoa[1])
            assert np.array_equal(rows[:, s], without[:, s])                  # pattern (0, 0) at that pulsar
            assert not np.array_equal(rows, without)


# ------------------------------------------------------------------ timing fit
def test_timing_fit_projects_the_injection():
    import torch
    from pta_replicator_b200 import _cabi
    b = _cgw_batch(3, ntoas=(65, 193, 1025))
    for i in range(b.n_psr):
        b.set_timing_model(i, poly=2, jumps="f")
    R = 8
    post0 = b.generate(R, seed=SEED)
    pre0 = b._generate(R, SEED, 0, None, None, None, 0, None, postfit=False).clone()
    b.set_cw_population(n_sources=3, log10_h0=-13.0, pphase="uniform")
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
    print(f"\n[cwpop] timing fit: max |(post-fit with - without) - fit(injection)| = {err:.3e} of {scale:.3e}")
    assert err <= 1e-12 * scale


# ------------------------------------------------------------------ end to end through the Fe-statistic
def test_fe_statistic_end_to_end_ng15_epoch():
    from pta_replicator_b200.engine import healpix_ring_centres
    from tests.test_gpu_fp_statistic import NF, _batch, _ng15
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=False, n_freqs=NF)
    b.set_fe_statistic(nside=8)
    sky = healpix_ring_centres(8)
    s_star, f_star = 300, 6
    lf = float(np.log10(b._fp["freqs"][f_star]))
    R = 4096

    def population(log10_h0, fixed_sky=True):
        b.set_cw_population(n_sources=1, log10_h0=log10_h0, log10_fgw=lf, log10_mc=9.2,
                            gwtheta=sky[s_star, 0] if fixed_sky else None, gwphi=sky[s_star, 1] if fixed_sky else None,
                            psrTerm=False)

    def signal_power(n):
        with_ = b.generate(n, seed=SEED)
        b.set_cw_population(None)
        rows = with_ - b.generate(n, seed=SEED)
        return 2.0 * b.fp_statistic_of(rows, maps=True)["Fe"][:, f_star, s_star]

    population(-14.0)
    ss0 = float(signal_power(256).mean())
    h = -14.0 + 0.5 * np.log10(100.0 / ss0)                # <s|s> scales as h0^2: mean <s|s> ~ 100
    population(h)
    ss = _np(signal_power(R))
    population(h)
    x = 2.0 * _np(b.fp_statistic(R, seed=SEED, maps=True)["Fe"][:, f_star, s_star])
    se = np.sqrt(np.mean(2.0 * (4 + 2 * ss)) / R)
    z = np.mean(x - 4 - ss) / se
    print(f"\n[cwpop] Fe end to end, R={R}: mean <s|s> {ss.mean():.2f}, mean(2Fe - 4 - <s|s>) {np.mean(x - 4 - ss):.3f}, "
          f"z = {z:.2f}")
    assert abs(z) < 4
    population(h + 0.5 * np.log10(30.0), fixed_sky=False)  # isotropic sky, loud: mean <s|s> ~ 3000 at the fixed sky
    am = _np(b.fp_statistic(1024, seed=SEED + 1)["Fp_argmax"])
    frac = float(np.mean(am == f_star))
    print(f"[cwpop] isotropic loud population: Fp_argmax == f* in {frac:.4f} of 1024 realizations")
    assert frac >= 0.99


# ------------------------------------------------------------------ removal and refusals
def test_removal_and_refusals():
    import torch
    fresh = _cgw_batch(3)
    ref = fresh.generate(8, seed=SEED)
    b = _cgw_batch(3)
    b.set_cw_population(n_sources=2)
    with_ = b.generate(8, seed=SEED)
    assert not torch.equal(with_, ref)
    with pytest.raises(ValueError):
        b.generate(8, inject=dict(z1=torch.zeros(8, b.ld), z2=torch.zeros(8, b.ld)))
    with pytest.raises(ValueError, match="generate"):
        b.generate_to_host(8, seed=SEED)
    b.set_cw_population(None)
    assert torch.equal(b.generate(8, seed=SEED), ref)
    with pytest.raises(ValueError):
        b.cw_population_params(8)
