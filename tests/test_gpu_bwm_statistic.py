"""GPU tests of the burst-with-memory search (``PulsarBatch.set_bwm_statistic`` -> ``ptar_fp_project`` on the whitened
ramps + ``ptar_bwm_sky`` + ``ptar_bwm_combine``): the device against the plan's statics in numpy on the device's own X^,
the maxima against the returned maps, bit-identity across chunking, real0 splits, outputs and paths (and of the Fp / Fe
outputs of the same batch), an edge sweep against an extended-precision evaluation of the same formula with guards past
every output, the chi^2_2 / chi^2_1 null laws, a coherent ``add_gw_memory`` injection and a single-pulsar ramp against the
dense oracle's matched-filter power, and the batch injection against the drop-in."""
import numpy as np
import pytest

from tests import bwm_oracle as BO
from tests import os_oracle as OO
from tests import reduction_reference as RR
from tests.test_bwm_statistic_cpu import bwm_of_layout, unpack_layout
from tests.test_gpu_fe_statistic import _check_maxima
from tests.test_gpu_fp_statistic import SEED, _models, _ng15
from tests.test_gpu_reduction_edges import _rows      # noise, zero, timing-model-like and sinusoid rows, cycling

pytestmark = pytest.mark.gpu

T = 100
KEYS = ("bwm_max", "bwm_argmax_t0", "bwm_argmax_sky", "bwm_t0max", "bwm_t0argmax", "bwm_strain", "bwm_pol", "bwm_fap",
        "psr_max", "psr_argmax_t0", "psr_slope", "psr_fap")
MAXIMA = ("bwm", "bwm_t0max", "bwm_t0argmax", "bwm_max", "bwm_argmax_t0", "bwm_argmax_sky")


def _batch(psrs, noise, gwb=True, tm=True, **bwm):
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise, gwb=gwb)
    if tm:
        for i in range(b.n_psr):
            b.set_timing_model(i, poly=2, jumps="f")
    b.set_bwm_statistic(**bwm)
    return b


def _layout(b):
    """The BWM statics as the device holds them, in the ``plan()["bwm"]`` keys ``unpack_layout`` reads."""
    d = b.compile()["bwm"]
    return dict(sqm=d["sqm"].cpu().numpy(), ant=d["ant"].cpu().numpy(), linv=d["linv"].cpu().numpy(), n_t0=d["n_t0"],
                n_sky=d["n_sky"])


def _check_pulsar_term(res, seen):
    """psr_* equal 1/2 amps^2 reduced over the seen epochs (first index on ties), slope amps / sqrt(m) there."""
    import torch
    X = res["amps"].cpu().numpy()
    bp = np.where(seen[None], 0.5 * X * X, -np.inf)
    arg = np.argmax(bp, axis=2)
    assert np.array_equal(res["psr_argmax_t0"].cpu().numpy(), arg)
    assert np.array_equal(res["psr_max"].cpu().numpy(), np.take_along_axis(bp, arg[..., None], 2)[..., 0])
    m = res["m"].cpu().numpy()
    xs = np.take_along_axis(X, arg[..., None], 2)[..., 0]
    assert np.array_equal(res["psr_slope"].cpu().numpy(), xs / np.sqrt(m[np.arange(m.shape[0])[None, :], arg]))
    # erfc(x) has relative condition number ~2x^2 + 1, and scipy's own evaluation (exp(-x^2) of a rounded x^2) errs by as
    # much: the two agree to a few (x^2 + 2) ulps, down to the subnormal range
    from scipy.special import erfc
    x = np.sqrt(res["psr_max"].cpu().numpy())
    ref = erfc(x)
    assert np.all(np.abs(res["psr_fap"].cpu().numpy() - ref) <= 8 * (x * x + 2) * 2.0**-53 * ref + 1e-300)
    assert res["psr_argmax_t0"].dtype == torch.int64


def test_device_matches_numpy_ng15_full():
    """ng15-full, T = 100, nside 8, 64 post-fit rows with maps and amps: B within 1e-10 max(1, B) of numpy on the
    device's X^ and the plan's statics; every maximum equals the map's; the pulsar term equals 1/2 X^^2 over the seen
    epochs; B <= 1/2 sum_a X^^2 (1 + 1e-12)."""
    import torch
    psrs, noise = _ng15()
    b = _batch(psrs, noise, n_epochs=T, nside=8)
    lay = _layout(b)
    S = lay["n_sky"]
    rows = b.generate(64, seed=SEED)
    res = b.bwm_statistic_of(rows, pulsars=True, maps=True)
    X = res["amps"].cpu().numpy()
    ref, _ = bwm_of_layout(lay, X)
    B = res["bwm"].cpu().numpy()
    err = float(np.max(np.abs(B - ref) / np.maximum(1.0, ref)))
    print(f"\n[bwm] device vs numpy, 64 ng15-full rows, T={T}, S={S}: max |dB| / max(1, B) {err:.1e}; bwm_max range "
          f"{float(res['bwm_max'].min()):.1f} .. {float(res['bwm_max'].max()):.1f}; seen {int(res['seen'].sum())}/"
          f"{res['seen'].numel()}; host statics {res['setup_s']:.2f} s")
    assert err <= 1e-10
    _check_maxima(res, S, MAXIMA)
    assert torch.equal(res["bwm_fap"], torch.exp(-res["bwm_max"]))
    _check_pulsar_term(res, res["seen"].cpu().numpy())
    assert np.all(B <= 0.5 * np.sum(X * X, axis=1)[:, :, None] * (1 + 1e-12))
    assert torch.all((res["bwm_pol"] >= 0) & (res["bwm_pol"] < np.pi)) and torch.all(res["bwm_strain"] >= 0)
    assert res["sky"].shape == (S, 2) and res["antenna"].shape == (b.n_psr, S, 2) and res["t0_mjd"].shape == (T,)


def test_bit_identity_across_chunks_real0_outputs_and_paths():
    import torch
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise, n_epochs=T, nside=8)
    R = 1024
    a = b.bwm_statistic(R, seed=SEED, chunk=1024, pulsars=True, maps=True)
    c = b.bwm_statistic(R, seed=SEED, chunk=256, pulsars=True, maps=True)
    lo = b.bwm_statistic(512, seed=SEED, real0=0, pulsars=True, maps=True)
    hi = b.bwm_statistic(512, seed=SEED, real0=512, pulsars=True, maps=True)
    bare = b.bwm_statistic(R, seed=SEED, chunk=256)
    for k in KEYS + ("amps", "bwm"):
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    for k in KEYS:
        assert torch.equal(a[k], bare[k]), k
    assert "bwm" not in bare and "amps" not in bare
    _check_maxima(a, int(a["sky"].shape[0]), MAXIMA)
    assert torch.equal(a["bwm_fap"], torch.exp(-a["bwm_max"]))
    # without a timing model the generated rows are the rows the statistic reduces
    b2 = _batch(psrs, noise, tm=False, n_epochs=T, nside=8)
    e = b2.bwm_statistic(R, seed=SEED, pulsars=True, maps=True)
    f = b2.bwm_statistic_of(b2.generate(R, seed=SEED), pulsars=True, maps=True)
    for k in KEYS + ("amps", "bwm"):
        assert torch.equal(e[k], f[k]), k
    # the Fp / Fe outputs of the batch are unchanged by the registration
    def fp_batch(bwm):
        x = PulsarBatch(psrs)
        synthetic.ng15_recipe(x, noise)
        for i in range(x.n_psr):
            x.set_timing_model(i, poly=2, jumps="f")
        x.set_fp_statistic(n_freqs=20)
        x.set_fe_statistic(nside=4)
        if bwm:
            x.set_bwm_statistic(n_epochs=T, nside=8)
        return x.fp_statistic(256, seed=SEED, pulsars=True, maps=True)
    p, q = fp_batch(False), fp_batch(True)
    for k in ("Fp", "Fp_max", "Fp_argmax", "fap", "amps", "Fe", "Fe_fmax", "Fe_fargmax", "Fe_max", "Fe_argmax_f",
              "Fe_argmax_sky"):
        assert torch.equal(p[k], q[k]), k


# (P, T, S, R): every pulsar count, epoch count, sky size and realization count of the sweep appears at least once
EDGE_CASES = [(2, 512, 33, 130), (3, 1, 768, 1025), (67, 511, 1, 33), (128, 3, 33, 1), (67, 2, 768, 130),
              (2, 3, 1, 1)]


def _edge_grid(b, T_, S):
    """T_ epochs inside the span every pulsar observes and S sky points: the HEALPix nside-8 centres for 768 on many
    pulsars, otherwise isotropic points; on 2 or 3 pulsars only points whose antenna patterns are far from parallel
    (|sin| of the angle between two pulsars' (F+, Fx) > 0.3, each of norm > 0.05), where M2 is well conditioned."""
    from pta_replicator_b200.engine import antenna_patterns, healpix_ring_centres
    from pta_replicator_b200 import orf
    lo = max(float(m.min()) for m in b.mjd) + 1.0
    hi = min(float(m.max()) for m in b.mjd) - 1.0
    t0 = np.linspace(lo, hi, T_ + 2)[1:-1]
    if S == 768 and b.n_psr > 3:
        return t0, healpix_ring_centres(8)
    rng = np.random.default_rng(11)
    cand = np.stack([np.arccos(rng.uniform(-1, 1, 8 * S + 64)), rng.uniform(0, 2 * np.pi, 8 * S + 64)], axis=1)
    if b.n_psr <= 3:
        locs = orf.psrlocs_from_pulsars(b.psrs)
        e = antenna_patterns(np.pi / 2 - locs[:, 1], locs[:, 0], cand)                   # [P, C, 2]
        nrm = np.linalg.norm(e, axis=2)
        sin = np.abs(e[0, :, 0] * e[1, :, 1] - e[0, :, 1] * e[1, :, 0]) / np.maximum(nrm[0] * nrm[1], 1e-300)
        cand = cand[(sin > 0.3) & np.all(nrm > 0.05, axis=0)]
    assert len(cand) >= S
    return t0, cand[:S]


@pytest.mark.parametrize("P,T_,S,R", EDGE_CASES)
def test_bwm_edges_against_extended_precision(P, T_, S, R):
    """Device B against the same formula in longdouble on the device's X^ and statics.  Bound, first order and rigorous
    for any summation order: with g = gamma_{P+16}, |dN2| <= g sum_a |e_a| |sqrt(m_a) X^_a|, |dy| <= g |L2^-1| (that
    sum), |dB| <= sum_i |y_i| |dy_i| + gamma_8 B.  The launches then go through the C ABI with guards past every output:
    nothing outside [R, T, S] / [R, T] / [R] / [R, P] moves."""
    import ctypes as C
    import torch
    from pta_replicator_b200 import _cabi
    ntoas = tuple((64, 65, 193, 1025)[j % 4] if P <= 3 else (64, 65, 193)[j % 3] for j in range(P))
    b = RR.edge_batch(ntoas, seed=P + S + T_)
    t0, sky = _edge_grid(b, T_, S)
    b.set_bwm_statistic(t0_mjd=t0, sky=sky)
    lay = _layout(b)
    rows = torch.from_numpy(_rows(b, R, seed=R + P)).to(b.device)
    res = b.bwm_statistic_of(rows, pulsars=True, maps=True)
    X = res["amps"].cpu().numpy()
    dev = res["bwm"].cpu().numpy()
    sub = np.unique(np.r_[0, np.arange(R)[:: max(1, R // 40)], R - 1])       # rows evaluated in extended precision
    ref, N2 = bwm_of_layout(lay, X[sub], dtype=np.longdouble)
    sq, ant, Li = unpack_layout(lay)
    B2 = np.einsum("asp,rat->rtsp", np.abs(ant), np.abs(X[sub] * sq[None]))
    g = RR.gamma(P + 16)
    dy = g * np.einsum("tsij,rtsj->rtsi", np.abs(Li), B2)
    _, _, Lil = unpack_layout(lay, np.longdouble)
    y = np.abs(np.einsum("tsij,rtsj->rtsi", Lil, N2)).astype(float)
    bound = np.sum(y * dy, axis=-1) + RR.gamma(8) * ref.astype(float) + 1e-300
    ratio = float(np.max(np.abs(dev[sub] - ref.astype(float)) / bound))
    print(f"\n[bwm edges] P={P} T={T_} S={S} R={R}: worst |dB| / bound {ratio:.3f}")
    assert ratio <= 1
    _check_maxima(res, S, MAXIMA)
    assert torch.equal(res["bwm_fap"], torch.exp(-res["bwm_max"]))
    _check_pulsar_term(res, res["seen"].cpu().numpy())
    st = b.compile()["bwm"]
    G = 4096
    amps = torch.zeros((R, P, st["ncol"]), dtype=torch.float64, device=b.device)
    amps[:, :, :T_] = res["amps"]
    f64, i64 = dict(dtype=torch.float64, device=b.device), dict(dtype=torch.int64, device=b.device)
    maps = torch.full((R * T_ * S + G,), -7.0, **f64)
    tmax = torch.full((R * T_ + G,), -7.0, **f64)
    targ = torch.full((R * T_ + G,), -7, **i64)
    L = _cabi.lib()
    bm = C.byref(st["bwm"])
    _cabi.check(L.ptar_bwm_sky(amps.data_ptr(), R, bm, tmax.data_ptr(), targ.data_ptr(), maps.data_ptr(),
                               _cabi.current_stream()), "ptar_bwm_sky")
    per_r = [torch.full((R + G,), -7.0, **f64), torch.full((R + G,), -7, **i64), torch.full((R + G,), -7, **i64)] + \
        [torch.full((R + G,), -7.0, **f64) for _ in range(3)]
    per_p = [torch.full((R * P + G,), -7.0, **f64), torch.full((R * P + G,), -7, **i64),
             torch.full((R * P + G,), -7.0, **f64), torch.full((R * P + G,), -7.0, **f64)]
    _cabi.check(L.ptar_bwm_combine(amps.data_ptr(), tmax.data_ptr(), targ.data_ptr(), R, bm,
                                   *(t.data_ptr() for t in per_r + per_p), _cabi.current_stream()), "ptar_bwm_combine")
    torch.cuda.synchronize()
    assert torch.all(maps[R * T_ * S:] == -7.0) and torch.all(tmax[R * T_:] == -7.0) and torch.all(targ[R * T_:] == -7)
    assert all(torch.all(t[R:] == -7) for t in per_r) and all(torch.all(t[R * P:] == -7) for t in per_p)
    assert torch.equal(maps[:R * T_ * S].view(R, T_, S), res["bwm"]) and torch.equal(tmax[:R * T_].view(R, T_), res["bwm_t0max"])
    for t, k in zip(per_r + per_p, ("bwm_max", "bwm_argmax_t0", "bwm_argmax_sky", "bwm_strain", "bwm_pol", "bwm_fap",
                                    "psr_max", "psr_argmax_t0", "psr_slope", "psr_fap")):
        assert torch.equal(t[:res[k].numel()].view(res[k].shape), res[k]), k


def test_null_law_ng15_full():
    """White + ECORR + RN with timing models, no GWB, P = the generating model: 2B ~ chi^2_2 at every cell and
    2Bp ~ chi^2_1 at every seen (pulsar, epoch) cell.  At 256 fixed cells of each the mean is within 5 standard errors of
    2 (1) and var / 4 (var / 2) within 1 +- 0.2 (the sd of the sample variance is 3.2 % for chi^2_2 and 4.0 % for
    chi^2_1 at R = 4096, so 0.2 is 5 sd or more)."""
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False, n_epochs=T, nside=8)
    R = 4096
    res = b.bwm_statistic(R, seed=SEED + 3, pulsars=True)
    lay = _layout(b)
    S = lay["n_sky"]
    rng = np.random.default_rng(5)
    cells = np.stack([rng.integers(0, T, 256), rng.integers(0, S, 256)], axis=1)
    X = res["amps"].cpu().numpy()
    sq, ant, Li = unpack_layout(lay)
    W = X[:, :, cells[:, 0]] * sq[:, cells[:, 0]][None]                         # [R, P, 256]
    N2 = np.einsum("acp,rac->rcp", ant[:, cells[:, 1]], W)
    y = np.einsum("cij,rcj->rci", Li[cells[:, 0], cells[:, 1]], N2)
    x = np.sum(y * y, axis=-1)                                                   # 2B
    z = (x.mean(axis=0) - 2.0) / np.sqrt(4.0 / R)
    v = x.var(axis=0, ddof=1) / 4
    seen = np.argwhere(res["seen"].cpu().numpy())
    pc = seen[rng.choice(len(seen), 256, replace=False)]
    xp = X[:, pc[:, 0], pc[:, 1]] ** 2                                          # 2Bp
    zp = (xp.mean(axis=0) - 1.0) / np.sqrt(2.0 / R)
    vp = xp.var(axis=0, ddof=1) / 2
    print(f"\n[bwm] null law R={R}, P={b.n_psr}: 2B z in [{z.min():.2f}, {z.max():.2f}], var/4 in [{v.min():.3f}, "
          f"{v.max():.3f}]; 2Bp z in [{zp.min():.2f}, {zp.max():.2f}], var/2 in [{vp.min():.3f}, {vp.max():.3f}]; mean "
          f"bwm_max {float(res['bwm_max'].mean()):.2f}")
    assert np.all(np.abs(z) < 5) and np.all(np.abs(v - 1) < 0.2)
    assert np.all(np.abs(zp) < 5) and np.all(np.abs(vp - 1) < 0.2)


def test_coherent_injection_ng15_epoch():
    """PulsarBatch.add_gw_memory at grid epoch k* and nside-8 pixel s*, psi = 0.3, strain scaled so that the dense
    oracle's <s|s> = 100: on the signal-only row 2B(k*, s*) = <s|s> within 1e-10 relative, the argmax is (k*, s*) and
    the strain and polarisation are recovered within 1e-8; with noise the mean of 2B(k*, s*) is 2 + <s|s> within 4
    standard errors."""
    import torch
    from pta_replicator_b200.engine import healpix_ring_centres
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=False, n_epochs=T, nside=8)
    t0 = b._bwm["t0_mjd"]
    sky = healpix_ring_centres(8)
    k_star, s_star, psi = 37, 300, 0.3
    src = dict(gwtheta=sky[s_star, 0], gwphi=sky[s_star, 1], bwm_pol=psi, t0_mjd=t0[k_star])
    models = _models(b)
    S = BO.statics(b, t0[k_star:k_star + 1], models=models)

    def row_of(h):
        d = b.memory_delays(h, **src)
        row = np.zeros(b.ld)
        for i in range(b.n_psr):
            row[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = d[i]
        return row

    from tests import fe_oracle as EO
    ss1 = EO.signal_power(b, S, row_of(1e-14), models=models)
    h = 1e-14 * float(np.sqrt(100.0 / ss1))                   # the ramp scales with the strain: <s|s> = 100
    row = row_of(h)
    ss = EO.signal_power(b, S, row, models=models)
    res = b.bwm_statistic_of(torch.from_numpy(row[None, :]).to(b.device), maps=True)
    b2 = 2.0 * float(res["bwm"][0, k_star, s_star])
    rel = abs(b2 - ss) / ss
    dh = abs(float(res["bwm_strain"][0]) - h) / h
    dpsi = abs(float(res["bwm_pol"][0]) - psi)
    print(f"\n[bwm] memory burst on ng15-epoch at (t0 {k_star}, s {s_star}): <s|s> {ss:.4f}, 2B {b2:.4f}, relative "
          f"{rel:.1e}; argmax (t0 {int(res['bwm_argmax_t0'][0])}, s {int(res['bwm_argmax_sky'][0])}); strain {h:.4e} "
          f"recovered to {dh:.1e}, psi to {dpsi:.1e}")
    assert rel <= 1e-10
    assert int(res["bwm_argmax_t0"][0]) == k_star and int(res["bwm_argmax_sky"][0]) == s_star
    assert dh <= 1e-8 and dpsi <= 1e-8
    b.add_gw_memory(h, **src)
    R = 4096
    X = b.bwm_statistic(R, seed=SEED + 5, pulsars=True)["amps"].cpu().numpy()
    lay = _layout(b)
    sq, ant, Li = unpack_layout(lay)
    N2 = np.einsum("ap,ra->rp", ant[:, s_star], X[:, :, k_star] * sq[:, k_star])
    y = N2 @ Li[k_star, s_star].T
    x = np.sum(y * y, axis=1)
    se = np.sqrt(2.0 * (2 + 2 * ss) / R)
    z = (x.mean() - (2 + ss)) / se
    print(f"[bwm] noise + burst, R={R}: mean 2B {x.mean():.3f} vs 2 + <s|s> = {2 + ss:.3f}, z = {z:.2f}")
    assert abs(z) < 4


def test_pulsar_term_injection():
    """A ramp of slope 3e-15 s/s in one pulsar at a grid epoch (set_deterministic): psr_max = <s|s> / 2 of that pulsar's
    dense oracle within 1e-10 relative, psr_slope the injected slope within 1e-8, at the injected epoch."""
    import torch
    psrs, noise = _ng15("epoch", npsr=8)
    b = _batch(psrs, noise, gwb=False, n_epochs=T, nside=1)
    a, k, slope = 5, 61, 3e-15
    t0 = b._bwm["t0_mjd"][k]
    models = _models(b)
    u = BO.ramps(b, a, [t0])[:, 0]
    s_tab = np.empty(b.ntoa[a])
    s_tab[b.order[a]] = slope * u
    b.set_deterministic(a, s_tab)
    row = np.zeros(b.ld)
    row[b.toa_off[a]:b.toa_off[a] + b.ntoa[a]] = b._det[a]                    # the delay as the batch holds it
    assert np.array_equal(b._det[a], slope * u)
    Pa = OO.dense_covariance(b, a)
    ss = float((slope * u) @ OO.c_matrix(Pa, (slope * u)[:, None], models[a])[:, 0])
    res = b.bwm_statistic_of(torch.from_numpy(row[None, :]).to(b.device), pulsars=True)
    pm, ps = float(res["psr_max"][0, a]), float(res["psr_slope"][0, a])
    print(f"\n[bwm] pulsar-term ramp in pulsar {a} at epoch {k}: <s|s>/2 {ss / 2:.4f}, psr_max {pm:.4f}, slope "
          f"{ps:.6e} vs {slope:.6e}; argmax epoch {int(res['psr_argmax_t0'][0, a])}")
    assert abs(pm - ss / 2) <= 1e-10 * ss / 2
    assert abs(ps - slope) <= 1e-8 * slope and int(res["psr_argmax_t0"][0, a]) == k
    others = [i for i in range(b.n_psr) if i != a]
    assert torch.all(res["psr_max"][0, others] == 0)


def test_batch_injection_matches_drop_in():
    """PulsarBatch.add_gw_memory adds to each pulsar, bit for bit, what the drop-in deterministic.add_gw_memory adds to
    that pulsar (table order, reordered to engine order)."""
    from pta_replicator_b200 import deterministic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, _ = _ng15("epoch", npsr=6)
    b = PulsarBatch(psrs)
    args = dict(strain=3.1e-14, gwtheta=1.1, gwphi=4.2, bwm_pol=0.7, t0_mjd=55555.25)
    d = b.memory_delays(**args)
    b.add_gw_memory(**args)
    for i, p in enumerate(psrs):
        deterministic.add_gw_memory(p, **args)
        ref = np.asarray(p.added_signals_time[f"{p.name}_gw_memory"].value)[b.order[i]]
        assert np.array_equal(d[i], ref), i
        assert np.array_equal(b._det[i], ref), i
        assert np.any(ref != 0) and np.any(ref == 0)
