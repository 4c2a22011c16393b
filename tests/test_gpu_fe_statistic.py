"""GPU tests of the Fe-statistic (``PulsarBatch.set_fe_statistic`` -> ``ptar_fe_sky`` + ``ptar_fe_combine`` after
``ptar_fp_project``): the device against the plan's statics in numpy on the device's own X^, the maxima against the
returned maps, bit-identity across chunking, real0 splits and paths (and of the Fp outputs with and without a sky grid),
an edge sweep against an extended-precision evaluation of the same formula, the chi^2_4 null law and an injected
``add_cgw`` source against the dense oracle's matched-filter power."""
import numpy as np
import pytest

from tests import fe_oracle as EO
from tests import fp_oracle as FO
from tests import reduction_reference as RR
from tests.test_fe_statistic_cpu import fe_of_layout
from tests.test_gpu_fp_statistic import SEED, _batch, _models, _ng15
from tests.test_gpu_reduction_edges import _rows      # noise, zero, timing-model-like and sinusoid rows, cycling

pytestmark = pytest.mark.gpu

NF = 100
FE_KEYS = ("Fe_fmax", "Fe_fargmax", "Fe_max", "Fe_argmax_f", "Fe_argmax_sky", "Fe")
FP_KEYS = ("Fp", "Fp_max", "Fp_argmax", "fap", "amps")
FE_MAXIMA = ("Fe", "Fe_fmax", "Fe_fargmax", "Fe_max", "Fe_argmax_f", "Fe_argmax_sky")


def _layout(b):
    """The Fe statics as the device holds them."""
    d = b.compile()["fp"]["fe"]
    return {k: d[k].cpu().numpy() for k in ("Lf", "ant", "linv")}, d["n_sky"]


def _check_maxima(res, S, names=FE_MAXIMA):
    """The maxima of a sky statistic equal those of its returned map exactly (first index on ties).  ``names``: the map
    [R, rows, S] (rows: frequencies or epochs), the per-row maximum over the sky and its argmax, the overall maximum and
    its row and sky indices."""
    import torch
    m, row_max, row_arg, top, top_row, top_sky = names
    assert torch.equal(res[row_max], res[m].max(dim=2).values)
    mp = res[m].cpu().numpy()
    assert np.array_equal(res[row_arg].cpu().numpy(), np.argmax(mp, axis=2))
    assert torch.equal(res[top], res[row_max].max(dim=1).values)
    flat = np.argmax(mp.reshape(mp.shape[0], -1), axis=1)                   # row-major: lower row, then lower s
    assert np.array_equal(res[top_row].cpu().numpy(), flat // S)
    assert np.array_equal(res[top_sky].cpu().numpy(), flat % S)
    assert int(res[row_arg].max()) < S and int(res[top_sky].max()) < S


def test_device_matches_numpy_ng15_full():
    """ng15-full, Nf = 100, nside 8, 64 post-fit rows with maps: Fe within 1e-10 max(1, Fe) of numpy on the device's X^ and
    the plan's statics; every maximum equals the map's; Fe_fmax <= Fp (1 + 1e-12)."""
    import torch
    psrs, noise = _ng15()
    b = _batch(psrs, noise, n_freqs=NF)
    b.set_fe_statistic(nside=8)
    lay, S = _layout(b)
    rows = b.generate(64, seed=SEED)
    res = b.fp_statistic_of(rows, pulsars=True, maps=True)
    ref, _ = fe_of_layout(lay["Lf"], lay["ant"], lay["linv"], b.n_psr, S, res["amps"].cpu().numpy())
    fe = res["Fe"].cpu().numpy()
    err = float(np.max(np.abs(fe - ref) / np.maximum(1.0, ref)))
    print(f"\n[fe] device vs numpy, 64 ng15-full rows, Nf={NF}, S={S}: max |dFe| / max(1, Fe) {err:.1e}; "
          f"Fe_max range {float(res['Fe_max'].min()):.1f} .. {float(res['Fe_max'].max()):.1f}; host statics "
          f"{res['fe_setup_s']:.2f} s")
    assert err <= 1e-10
    _check_maxima(res, S)
    assert torch.all(res["Fe_fmax"] <= res["Fp"] * (1 + 1e-12))
    assert res["sky"].shape == (S, 2) and res["antenna"].shape == (b.n_psr, S, 2)
    assert res["Fe_fargmax"].dtype == torch.int64 and res["Fe_argmax_f"].dtype == torch.int64


def test_bit_identity_across_chunks_real0_paths_and_registration():
    import torch
    psrs, noise = _ng15(npsr=24)
    b = _batch(psrs, noise, n_freqs=NF)
    b.set_fe_statistic(nside=8)
    R = 1024
    a = b.fp_statistic(R, seed=SEED, chunk=1024, pulsars=True, maps=True)
    c = b.fp_statistic(R, seed=SEED, chunk=256, pulsars=True, maps=True)
    lo = b.fp_statistic(512, seed=SEED, real0=0, pulsars=True, maps=True)
    hi = b.fp_statistic(512, seed=SEED, real0=512, pulsars=True, maps=True)
    nomap = b.fp_statistic(R, seed=SEED, chunk=256)
    for k in FE_KEYS + FP_KEYS:
        assert torch.equal(a[k], c[k]), k
        assert torch.equal(a[k], torch.cat([lo[k], hi[k]])), k
    for k in FE_KEYS[:-1] + FP_KEYS[:-1]:
        assert torch.equal(a[k], nomap[k]), k
    assert "Fe" not in nomap
    _check_maxima(a, int(a["sky"].shape[0]))
    # the Fp outputs do not change when a sky grid is registered
    plain = _batch(psrs, noise, n_freqs=NF)
    p = plain.fp_statistic(R, seed=SEED, pulsars=True)
    for k in FP_KEYS:
        assert torch.equal(a[k], p[k]), k
    assert "Fe_max" not in p
    with pytest.raises(ValueError, match="set_fe_statistic"):
        plain.fp_statistic(8, maps=True)
    # without a timing model the generated rows are the rows the statistic reduces
    b2 = _batch(psrs, noise, tm=False, n_freqs=NF)
    b2.set_fe_statistic(nside=8)
    e = b2.fp_statistic(R, seed=SEED, maps=True)
    f = b2.fp_statistic_of(b2.generate(R, seed=SEED), maps=True)
    for k in FE_KEYS + FP_KEYS[:-1]:
        assert torch.equal(e[k], f[k]), k


# (P, S, Nf, R): every pulsar count, sky size, frequency count and realization count of the sweep appears at least once
EDGE_CASES = [(2, 1, 256, 130), (3, 12, 1, 1025), (67, 768, 100, 33), (128, 33, 1, 1), (67, 3072, 1, 130),
              (2, 3072, 100, 1)]
EDGE_SKY_SEED = 11


def _edge_sky(S, b):
    """S sky points: the HEALPix centres for 768 and 3072, otherwise isotropic points; on 2 or 3 pulsars, points where M4
    has lambda_min / lambda_max > 1e-11 at every frequency (M4 is singular where the antenna patterns are parallel, and a
    pulsar of a few TOAs can make M_a(f) itself nearly singular)."""
    from pta_replicator_b200.engine import antenna_patterns, healpix_ring_centres
    from pta_replicator_b200 import orf
    if S in (768, 3072) and b.n_psr > 3:
        return healpix_ring_centres(int(round(np.sqrt(S / 12))))
    rng = np.random.default_rng(EDGE_SKY_SEED)
    cand = np.stack([np.arccos(rng.uniform(-1, 1, 4 * S + 64)), rng.uniform(0, 2 * np.pi, 4 * S + 64)], axis=1)
    if b.n_psr <= 3:
        locs = orf.psrlocs_from_pulsars(b.psrs)
        e = antenna_patterns(np.pi / 2 - locs[:, 1], locs[:, 0], cand)                  # [P, C, 2]
        M = b.plan()["fp"]["M"]                                                          # [P, Nf, 2, 2]
        M4 = np.einsum("asp,asq,afcd->sfpcqd", e, e, M).reshape(len(cand), M.shape[1], 4, 4)
        ev = np.linalg.eigvalsh(M4)
        cand = cand[np.all(ev[..., 0] > 1e-11 * ev[..., 3], axis=1)]
    assert len(cand) >= S
    return cand[:S]


@pytest.mark.parametrize("P,S,nf,R", EDGE_CASES)
def test_fe_edges_against_extended_precision(P, S, nf, R):
    """Device Fe against the same formula in longdouble on the device's X^ and statics.  Bound, first order and rigorous
    for any summation order: with g = gamma_{P+16}, |dN4| <= g sum_a |e_a| (x) |N|_a (|N|_a = |l11 x0|, |l21 x0| + |l22 x1|),
    |dy| <= g |L4^-1| (sum_a |e_a| (x) |N|_a), |dFe| <= sum_i |y_i| |dy_i| + gamma_8 Fe.  No argmax >= S; the map is
    written exactly on [R, Nf, S] (a guard past it stays untouched)."""
    import ctypes as C
    import torch
    from pta_replicator_b200 import _cabi
    ntoas = tuple(RR.EDGE_NTOAS[(3 * j) % len(RR.EDGE_NTOAS)] if P <= 3 else (64, 65, 193)[j % 3] for j in range(P))
    b = RR.edge_batch(ntoas, seed=P + S)
    b.set_fp_statistic(n_freqs=nf)
    b.set_fe_statistic(sky=_edge_sky(S, b))
    lay, S_ = _layout(b)
    assert S_ == S
    rows = torch.from_numpy(_rows(b, R, seed=R + P)).to(b.device)
    res = b.fp_statistic_of(rows, pulsars=True, maps=True)
    X = res["amps"].cpu().numpy()
    dev = res["Fe"].cpu().numpy()
    sub = np.unique(np.r_[0, np.arange(R)[:: max(1, R // 40)], R - 1])       # rows evaluated in extended precision
    ref, ant = fe_of_layout(lay["Lf"], lay["ant"], lay["linv"], P, S, X[sub], dtype=np.longdouble)
    # the bound, in fp64 on absolute values
    Xa = np.abs(X[sub])
    L = np.abs(lay["Lf"]).transpose(1, 0, 2)[None]
    Nabs = np.stack([L[..., 0] * Xa[..., 0], L[..., 1] * Xa[..., 0] + L[..., 2] * Xa[..., 1]], axis=-1)
    B4 = np.einsum("asp,rafc->rfspc", np.abs(ant.astype(float)), Nabs).reshape(len(sub), nf, S, 4)
    Li = np.zeros((nf, S, 4, 4))
    Li[..., np.tril_indices(4)[0], np.tril_indices(4)[1]] = np.abs(lay["linv"][:, :S])
    Li_signed = np.zeros((nf, S, 4, 4), dtype=np.longdouble)
    Li_signed[..., np.tril_indices(4)[0], np.tril_indices(4)[1]] = lay["linv"][:, :S]
    g = RR.gamma(P + 16)
    dy = g * np.einsum("fsij,rfsj->rfsi", Li, B4)
    # |y| from the extended-precision evaluation: recompute y in longdouble
    Xl = X[sub].astype(np.longdouble)
    Ll = lay["Lf"].astype(np.longdouble).transpose(1, 0, 2)[None]
    Nl = np.stack([Ll[..., 0] * Xl[..., 0], Ll[..., 1] * Xl[..., 0] + Ll[..., 2] * Xl[..., 1]], axis=-1)
    N4 = np.einsum("asp,rafc->rfspc", ant.astype(np.longdouble), Nl).reshape(len(sub), nf, S, 4)
    y = np.abs(np.einsum("fsij,rfsj->rfsi", Li_signed, N4)).astype(float)
    bound = np.sum(y * dy, axis=-1) + RR.gamma(8) * ref.astype(float) + 1e-300
    ratio = float(np.max(np.abs(dev[sub] - ref.astype(float)) / bound))
    print(f"\n[fe edges] P={P} S={S} Nf={nf} R={R}: worst |dFe| / bound {ratio:.3f}")
    assert ratio <= 1
    _check_maxima(res, S)
    # the same launch through the C ABI with guards past every output: nothing outside [R, Nf, S] / [R, Nf] / [R] moves
    st = b.compile()["fp"]["fe"]
    G = 4096
    amps = res["amps"].contiguous()
    maps = torch.full((R * nf * S + G,), -7.0, dtype=torch.float64, device=b.device)
    fmax = torch.full((R * nf + G,), -7.0, dtype=torch.float64, device=b.device)
    farg = torch.full((R * nf + G,), -7, dtype=torch.int64, device=b.device)
    L_ = _cabi.lib()
    _cabi.check(L_.ptar_fe_sky(amps.data_ptr(), R, C.byref(st["model"]), fmax.data_ptr(), farg.data_ptr(), maps.data_ptr(),
                               _cabi.current_stream()), "ptar_fe_sky")
    torch.cuda.synchronize()
    assert torch.all(maps[R * nf * S:] == -7.0) and torch.all(fmax[R * nf:] == -7.0) and torch.all(farg[R * nf:] == -7)
    assert torch.equal(maps[:R * nf * S].view(R, nf, S), res["Fe"]) and torch.equal(fmax[:R * nf].view(R, nf), res["Fe_fmax"])


def test_null_law_ng15_full():
    """White + ECORR + RN with timing models, no GWB, P = the generating model: 2Fe ~ chi^2_4 at every cell.  At 256 fixed
    cells the mean of 2Fe is within 5 standard errors of 4 and var / 8 within 1 +- 0.2 (the sd of the sample variance of
    chi^2_4 is 3.5 % at R = 4096, so 0.2 is 5.7 sd); Fe_fmax >= every cell of its frequency."""
    import torch
    psrs, noise = _ng15()
    b = _batch(psrs, noise, gwb=False, n_freqs=NF)
    b.set_fe_statistic(nside=8)
    R = 4096
    res = b.fp_statistic(R, seed=SEED + 3, maps=True)
    S = int(res["sky"].shape[0])
    rng = np.random.default_rng(5)
    cells = np.stack([rng.integers(0, NF, 256), rng.integers(0, S, 256)], axis=1)
    x = 2.0 * res["Fe"][:, cells[:, 0], cells[:, 1]].cpu().numpy()
    mean, var = x.mean(axis=0), x.var(axis=0, ddof=1)
    z = (mean - 4.0) / np.sqrt(8.0 / R)
    print(f"\n[fe] null law R={R}, P={b.n_psr}, 256 cells: z of mean 2Fe in [{z.min():.2f}, {z.max():.2f}], var / 8 in "
          f"[{(var / 8).min():.3f}, {(var / 8).max():.3f}]; mean Fe_max {float(res['Fe_max'].mean()):.2f}")
    assert np.all(np.abs(z) < 5)
    assert np.all(np.abs(var / 8 - 1) < 0.2)
    assert torch.all(res["Fe_fmax"][:, :, None] >= res["Fe"])
    assert torch.all(res["Fe_fmax"] <= res["Fp"] * (1 + 1e-12))


def test_injected_source_ng15_epoch():
    """An add_cgw source (psrTerm=False, evolve=False) at an nside-8 pixel and grid frequency index 6 lies in the 4-column
    span: 2Fe of the signal-only row at (f*, s*) equals the dense oracle's <s|s> and 2Fp(f*) within 1e-10, and the argmax
    is (f*, s*); with noise plus the source at <s|s> ~ 100, mean 2Fe(f*, s*) = 4 + <s|s> within 4 standard errors."""
    import torch
    from pta_replicator_b200.engine import healpix_ring_centres
    psrs, noise = _ng15("epoch")
    b = _batch(psrs, noise, gwb=False, n_freqs=NF)
    b.set_fe_statistic(nside=8)
    sky = healpix_ring_centres(8)
    s_star, f_star = 300, 6
    fgw = b._fp["freqs"][f_star]
    src = dict(gwtheta=sky[s_star, 0], gwphi=sky[s_star, 1], mc=10**9.2, fgw=fgw, phase0=0.7, psi=0.4, inc=1.0,
               psrTerm=False, evolve=False, phase_approx=False)
    S = FO.statics(b, b._fp["freqs"], models=_models(b))

    def row_of(dist):
        d = b.cgw_delays(dist=dist, **src)
        row = np.zeros(b.ld)
        for i in range(b.n_psr):
            row[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = d[i]
        return row

    ss1 = EO.signal_power(b, S, row_of(1.0), models=_models(b))
    dist = float(np.sqrt(ss1 / 100.0))                        # residuals scale as 1 / dist: <s|s> = 100
    row = row_of(dist)
    ss = EO.signal_power(b, S, row, models=_models(b))
    res = b.fp_statistic_of(torch.from_numpy(row[None, :]).to(b.device), maps=True)
    fe2 = 2.0 * float(res["Fe"][0, f_star, s_star])
    fp2 = 2.0 * float(res["Fp"][0, f_star])
    rel = max(abs(fe2 - ss) / ss, abs(fp2 - ss) / ss)
    print(f"\n[fe] CW on ng15-epoch at (f {f_star}, s {s_star}): <s|s> {ss:.4f}, 2Fe {fe2:.4f}, 2Fp {fp2:.4f}, worst "
          f"relative {rel:.1e}; argmax (f {int(res['Fe_argmax_f'][0])}, s {int(res['Fe_argmax_sky'][0])})")
    assert rel <= 1e-10
    assert int(res["Fe_argmax_f"][0]) == f_star and int(res["Fe_argmax_sky"][0]) == s_star
    b.add_cgw(dist=dist, **src)
    R = 4096
    x = 2.0 * b.fp_statistic(R, seed=SEED + 5, maps=True)["Fe"][:, f_star, s_star].cpu().numpy()
    se = np.sqrt(2.0 * (4 + 2 * ss) / R)
    z = (x.mean() - (4 + ss)) / se
    print(f"[fe] noise + source, R={R}: mean 2Fe {x.mean():.3f} vs 4 + <s|s> = {4 + ss:.3f}, z = {z:.2f}")
    assert abs(z) < 4
