"""GPU tests of the sine-Gaussian burst search (``PulsarBatch.set_burst_statistic`` -> ``ptar_fp_project`` (z) +
``ptar_burst_ninv`` + ``ptar_burst_project`` + ``ptar_fe_sky`` per group + ``ptar_burst_reduce``): the device amplitudes at
edge shapes against an extended-precision evaluation of the factored formula and against ``ptar_fp_project`` on the
dense oracle's whitened columns, the reductions against the maps, the coherent bound, noise-free ``add_burst`` and
``add_noise_transient`` injections against <s|s>, the chi^2_4 / chi^2_2 noise means, bit-identity across chunking, real0
splits, paths and maps, the batch ``add_burst`` against the drop-in, and the kernels' ptxas resources."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from tests import burst_oracle as UO

pytestmark = pytest.mark.gpu

SEED = 20261017
KEYS = ("B_max", "argmax_template", "argmax_sky", "fap", "amp", "B_template", "B_template_sky", "Bt_max",
        "argmax_template_psr", "fap_psr")


def _pulsars(P, nep=40, seed=3, shared=True, single=False):
    """P synthetic pulsars; with ``shared`` every pulsar observes the same epochs (3-6 sub-band TOAs within 1 s), so
    every template inside the span is seen by every pulsar; with ``single`` the last pulsar has one TOA per epoch."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    ep = np.sort(rng.uniform(53000.0, 58800.0, nep))
    out = []
    for j in range(P):
        if not shared:
            ep = np.sort(rng.uniform(53000.0, 58800.0, nep))
        nsub = rng.integers(3, 7, nep) if not (single and j == P - 1) else np.ones(nep, dtype=np.int64)
        mjd = np.concatenate([e + rng.uniform(0, 0.9, k) / 86400.0 for e, k in zip(ep, nsub)])
        be = np.concatenate([[("A", "B", "C")[q % 3]] * k for q, k in enumerate(nsub)])
        p = pulsar_from_arrays(f"G{j}", {"RAJ": float(rng.uniform(0, 24)), "DECJ": float(rng.uniform(-80, 80))},
                               mjd.astype(np.longdouble), rng.uniform(0.2, 2.0, mjd.size), flags=[{"f": f} for f in be])
        make_ideal(p)
        out.append(p)
    return out


def _batch(psrs, tm=True, red=True, coarsegrain=1.0 / 86400.0):
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(psrs)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.1, log10_equad=-6.5)
        b.set_ecorr(i, -6.3, coarsegrain=coarsegrain)
        if red:
            b.set_red(i, -13.8 - 0.01 * i, 3.5, components=10)
        if tm:
            b.set_timing_model(i, poly=2, jumps="f")
    return b


def _bank(b, J, seed=0):
    rng = np.random.default_rng(seed)
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    Tspan = (last - first) * 86400
    return (rng.uniform(first + 0.1 * (last - first), last - 0.1 * (last - first), J), rng.uniform(2.0, 25.0, J) / Tspan,
            rng.choice([4.0, 8.0], J))


def _rows(b, R, seed=1, poison=True):
    """Noise-level rows [R, ld] with NaN in every alignment slot (``poison``): no kernel may read them."""
    import torch
    rows = np.random.default_rng(seed).standard_normal((R, b.ld)) * 1e-6
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    rows[:, ~live] = np.nan if poison else 0.0
    return rows, torch.from_numpy(rows).to(b.device)


def _device_amps(b, rows_d):
    """X^ [R, P, J, 2] of the device: z, N^-1 r and every group's ptar_burst_project through the C ABI."""
    import torch
    from pta_replicator_b200 import _cabi
    st = b.compile()["burst"]
    L, R, P, J, G = _cabi.lib(), rows_d.shape[0], b.n_psr, st["n_tmpl"], _cabi.BURST_GROUP
    z = torch.full((R * P * st["n_zc"],), np.nan, dtype=torch.float64, device=b.device)
    y = torch.full((R, b.ld), np.nan, dtype=torch.float64, device=b.device)
    _cabi.check(L.ptar_fp_project(rows_d.data_ptr(), b.ld, R, C.byref(st["model"]), z.data_ptr(), None), "fp_project")
    _cabi.check(L.ptar_burst_ninv(rows_d.data_ptr(), b.ld, R, C.byref(st["burst"]), y.data_ptr(), None), "burst_ninv")
    out = np.empty((R, P, J, 2))
    for g in range(0, J, G):
        jg = min(G, J - g)
        a = torch.full((R * P * 2 * jg + 64,), np.nan, dtype=torch.float64, device=b.device)   # + a guard past the end
        _cabi.check(L.ptar_burst_project(y.data_ptr(), b.ld, R, z.data_ptr(), C.byref(st["burst"]), g // G, a.data_ptr(),
                                         None), "burst_project")
        torch.cuda.synchronize()
        ah = a.cpu().numpy()
        assert np.all(np.isnan(ah[R * P * 2 * jg:]))
        out[:, :, g:g + jg] = ah[:R * P * 2 * jg].reshape(R, P, jg, 2)
    return out


def _dense_fp(b, pb, S, rows_d):
    """X^ [R, P, J, 2] of ``ptar_fp_project`` run on the oracle's dense whitened columns P_a^-1 W_j L^-T (0 unseen), 256
    templates (PTAR_FP_MAX_FREQ) at a time."""
    import torch
    from pta_replicator_b200 import _cabi
    from pta_replicator_b200.engine import FP_CB, _put_columns
    J, R = pb["n_tmpl"], rows_d.shape[0]
    out = np.empty((R, b.n_psr, J, 2))
    for g in range(0, J, 256):
        jj = np.arange(g, min(J, g + 256))
        lay = b._fp_layout(len(jj))
        for i in range(b.n_psr):
            Ca = S["C"][i].reshape(b.ntoa[i], J, 2)[:, jj]
            seen = S["seen"][i][jj]
            L = np.linalg.cholesky(np.where(seen[:, None, None], S["M"][i][jj], np.eye(2)))
            Wt = np.zeros((b.ntoa[i], lay["n_cb"] * FP_CB))
            c0 = Ca[:, :, 0] / L[:, 0, 0]
            Wt[:, 0:2 * len(jj):2] = np.where(seen, c0, 0)
            Wt[:, 1:2 * len(jj):2] = np.where(seen, (Ca[:, :, 1] - L[:, 1, 0] * c0) / L[:, 1, 1], 0)
            _put_columns(lay["Ct"], b.toa_off[i], Wt)
        m, keep = b._fp_model(lay)
        amps = torch.empty(R * b.n_psr * 2 * len(jj), dtype=torch.float64, device=b.device)
        _cabi.check(_cabi.lib().ptar_fp_project(rows_d.data_ptr(), b.ld, R, C.byref(m), amps.data_ptr(), None),
                    "fp_project")
        out[:, :, jj] = amps.cpu().numpy().reshape(R, b.n_psr, len(jj), 2)
    return out


# (pulsars, templates, realizations, shared epochs, ECORR coarsegrain [days]): P = 2 and 128, J = 1, 256 and 257 (a group
# boundary), NR not a multiple of 64, ECORR runs of one TOA and runs of ~100 TOAs (longer than a 64-TOA chunk, crossing
# chunk boundaries), and a large bank of 1100 templates (five groups)
EDGES = [(2, 1, 5, True, 1.0 / 86400), (4, 257, 70, True, 2500.0), (128, 256, 3, True, 1.0 / 86400),
         (3, 40, 130, False, 2500.0), (3, 1100, 70, True, 1.0 / 86400)]


@pytest.mark.parametrize("P,J,R,shared,cg", EDGES)
def test_device_amps_match_references(P, J, R, shared, cg):
    b = _batch(_pulsars(P, shared=shared), coarsegrain=cg)
    t0, f0, Q = _bank(b, J)
    if J > 1:   # one window over the whole span
        t0[0], f0[0], Q[0] = 0.5 * (min(m.min() for m in b.mjd) + max(m.max() for m in b.mjd)), 1.0 / (6000 * 86400), 8.0
    b.set_burst_statistic(t0_mjd=t0, f0=f0, Q=Q, nside=1)
    pb = b.plan()["burst"]
    if cg > 1:
        assert pb["run_len"].max() > 64
    _check_amps(b, pb, R)


def test_device_amps_single_toa_windows():
    """Sub-second templates centred in observing epochs: the last pulsar has one TOA per epoch, so its windows hold a
    single TOA (unseen: X^ = 0) beside windows of 3-6 TOAs in the others, with no timing model or red noise to absorb
    them; and 20 templates of the span."""
    b = _batch(_pulsars(6, seed=8, single=True), tm=False, red=False)
    t0, f0, Q = _bank(b, 20)
    m = np.sort(b.mjd[0])
    first = np.flatnonzero(np.r_[True, np.diff(m) > 1e-3])
    ep = np.array([m[a:z].mean() for a, z in zip(first, np.r_[first[1:], len(m)])])[5:25]   # mid-epoch times
    tau = 0.25                                                          # s: the window spans +- 1.5 s, the epoch 0.9 s
    b.set_burst_statistic(t0_mjd=np.r_[t0, ep], f0=np.r_[f0, np.full(len(ep), 4.0 / (2 * np.pi * tau))],
                          Q=np.r_[Q, np.full(len(ep), 4.0)], nside=1)
    pb = b.plan()["burst"]
    width = pb["win"][..., 1] - pb["win"][..., 0]
    assert np.all(width[-1, :len(ep)] == 1) and not pb["seen"][-1, :len(ep)].any()
    assert np.all(width[:-1, :len(ep)] >= 3) and pb["seen"][:-1, :len(ep)].all()
    _check_amps(b, pb, 70)


def _check_amps(b, pb, R):
    rows, rows_d = _rows(b, R)
    got = _device_amps(b, rows_d)
    _, ref = UO.emulate(b, pb, np.nan_to_num(rows, nan=0.0), dtype=np.longdouble)
    ref = ref.astype(np.float64)
    d_ext = float(np.max(np.abs(got - ref)))
    S = UO.statics(b, pb["templates"], models=_models(b) if b._tm is not None else None)
    dense = _dense_fp(b, pb, S, rows_d)
    d_dense = float(np.max(np.abs(got - dense)))
    print(f"\n[burst amps] P={b.n_psr} J={pb['n_tmpl']} R={R}: |X^ - longdouble| {d_ext:.1e}, "
          f"|X^ - fp_project(dense)| {d_dense:.1e}")
    # X^ ~ N(0, 1): the fp64 sums over <= 10^3 TOAs and the rank-~70 H^T z cancellation leave ~1e-12 absolute
    assert d_ext < 1e-9 and d_dense < 1e-8
    assert np.all(got[:, ~pb["seen"]] == 0)


def _models(b):
    from tests import timing_oracle as TO
    out = []
    for i, p in enumerate(b.psrs):
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        out.append(TO.timing_design_matrix(t, 2, [f.get("f") for f in p.toas.table["flags"]])[b.order[i]])
    return out


def _check_reductions(res, seen, pulsars=True):
    B, Bt = res["B"].cpu().numpy(), res["Bt"].cpu().numpy()
    R, J, S = B.shape
    flat = B.reshape(R, -1)
    arg = np.argmax(flat, axis=1)
    assert np.array_equal(res["B_max"].cpu().numpy(), flat[np.arange(R), arg])
    assert np.array_equal(res["argmax_template"].cpu().numpy(), arg // S)
    assert np.array_equal(res["argmax_sky"].cpu().numpy(), arg % S)
    assert np.array_equal(res["B_template"].cpu().numpy(), B.max(axis=2))
    assert np.array_equal(res["B_template_sky"].cpu().numpy(), np.argmax(B, axis=2))
    bt = np.where(seen[None], Bt, -np.inf)
    assert np.array_equal(res["Bt_max"].cpu().numpy(), bt.max(axis=2))
    assert np.array_equal(res["argmax_template_psr"].cpu().numpy(), np.argmax(bt, axis=2))
    Bm = res["B_max"].cpu().numpy()
    assert np.allclose(res["fap"].cpu().numpy(), np.exp(-Bm) * (1 + Bm), rtol=1e-14, atol=0)
    assert np.allclose(res["fap_psr"].cpu().numpy(), np.exp(-bt.max(axis=2)), rtol=1e-14, atol=0)
    # B <= 1/2 sum_a |X^_a|^2 at every cell
    assert np.all(B <= Bt.sum(axis=1)[:, :, None] * (1 + 1e-12))


def test_noise_free_injections_and_reductions():
    import torch
    b = _batch(_pulsars(5))
    # 300 templates: the injected cell j = 280 lies in the second group of PTAR_BURST_GROUP
    b.set_burst_statistic(*_bank(b, 300, seed=5), nside=2)
    st = b.compile()["burst"]
    tm, sky = st["out"]["templates"].cpu().numpy(), st["out"]["sky"].cpu().numpy()
    j, s = 280, 17
    t0, f0, Q = tm[j, 0] * 86400, tm[j, 1], tm[j, 2]
    tau = Q / (2 * np.pi * f0)
    a = np.array([2e-7, -1e-7, 0.5e-7, 1.5e-7])

    def g(t):
        return np.exp(-((t - t0) / tau) ** 2)

    def c(t):
        return np.cos(2 * np.pi * f0 * (t - t0))

    def sn(t):
        return np.sin(2 * np.pi * f0 * (t - t0))

    b.add_burst(sky[s, 0], sky[s, 1], lambda t: a[0] * g(t) * c(t) + a[1] * g(t) * sn(t),
                lambda t: a[2] * g(t) * c(t) + a[3] * g(t) * sn(t))
    row = np.zeros(b.ld)
    for i in range(b.n_psr):
        row[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = b._det[i]
    rows = torch.from_numpy(np.tile(row, (4, 1))).to(b.device)
    res = b.burst_statistic_of(rows, pulsars=True, maps=True)
    pb = b.plan()["burst"]
    ant = b._antenna_patterns(sky)
    # <s|s> = sum_a c_a^T M_a c_a with s_a = W_j c_a, c_a = -(F+ (a0, a1) + Fx (a2, a3))
    ca = -(ant[:, s, 0:1] * a[None, :2] + ant[:, s, 1:2] * a[None, 2:])
    ss = float(np.einsum("ai,aij,aj->", ca, pb["M"][:, j], ca))
    B = res["B"].cpu().numpy()
    print(f"\n[burst injection] 2B / <s|s> - 1 = {2 * B[0, j, s] / ss - 1:.1e}, amp {res['amp'][0].cpu().numpy()} vs {a}")
    assert abs(2 * B[0, j, s] / ss - 1) < 1e-9
    assert int(res["argmax_template"][0]) == j and int(res["argmax_sky"][0]) == s
    assert np.allclose(res["amp"][0].cpu().numpy(), a, rtol=1e-6, atol=1e-8 * np.abs(a).max())
    _check_reductions(res, pb["seen"])
    # a noise transient in pulsar 3 only: Bt_3 = 1/2 <s|s>_3 at template j and amp_psr recovers (b0, b1)
    b2 = _batch(b.psrs)
    b2.set_burst_statistic(t0_mjd=tm[:, 0], f0=tm[:, 1], Q=tm[:, 2], nside=2)
    bw = np.array([3e-7, -2e-7])
    b2.add_noise_transient(3, lambda t: bw[0] * g(t) * c(t) + bw[1] * g(t) * sn(t))
    row = np.zeros(b2.ld)
    row[b2.toa_off[3]:b2.toa_off[3] + b2.ntoa[3]] = b2._det[3]
    res = b2.burst_statistic_of(torch.from_numpy(np.tile(row, (4, 1))).to(b2.device), pulsars=True, maps=True)
    M3 = b2.plan()["burst"]["M"][3, j]
    bt = float(res["Bt"][0, 3, j])
    assert abs(2 * bt / float(bw @ M3 @ bw) - 1) < 1e-9 and int(res["argmax_template_psr"][0, 3]) == j
    assert np.allclose(res["amp_psr"][0, 3].cpu().numpy(), bw, rtol=1e-6, atol=1e-8 * np.abs(bw).max())


def test_noise_means_and_determinism():
    import torch
    b = _batch(_pulsars(6))
    b.set_burst_statistic(nside=1)
    R = 512
    res = b.burst_statistic(R, seed=SEED, maps=True, pulsars=True)
    pb = b.plan()["burst"]
    B, Bt = res["B"].cpu().numpy(), res["Bt"].cpu().numpy()
    m4 = float(np.mean(2 * B))
    m2 = float(np.mean(2 * Bt[:, pb["seen"]]))
    print(f"\n[burst null] mean 2B = {m4:.3f} (chi^2_4: 4), mean 2Bt = {m2:.3f} (chi^2_2: 2), J = {pb['n_tmpl']}")
    # per cell the mean of R draws has sd sqrt(8 / R) = 0.125 (2B) and sqrt(4 / R) = 0.088 (2Bt); cells are correlated, so
    # the bound is 3 sd of one cell
    assert abs(m4 - 4) < 0.375 and abs(m2 - 2) < 0.27
    _check_reductions(res, pb["seen"])
    # bit-identity: chunk, real0 split, nreal, maps and pulsars off, and the rows path
    a = b.burst_statistic(16, seed=SEED, chunk=16)
    for other in (b.burst_statistic(16, seed=SEED, chunk=4),
                  {k: torch.cat([x[k], y[k]]) for x, y in [(b.burst_statistic(8, seed=SEED),
                                                           b.burst_statistic(8, seed=SEED, real0=8))] for k in KEYS}):
        for k in KEYS:
            assert torch.equal(a[k], other[k]), k
    for k in KEYS:
        assert torch.equal(a[k], res[k][:16]), k
    bn = _batch(b.psrs, tm=False)
    bn.set_burst_statistic(nside=1)
    x = bn.burst_statistic(12, seed=SEED)
    rows = bn.generate(12, seed=SEED)
    y = bn.burst_statistic_of(rows, maps=True)
    for k in KEYS:
        assert torch.equal(x[k], y[k]), k


def test_batch_add_burst_matches_drop_in(monkeypatch):
    from pta_replicator_b200 import deterministic
    psrs = _pulsars(3, shared=False)
    b = _batch(psrs)
    t0 = float(np.median(b.mjd[0])) * 86400

    def hp(t):
        return 1e-7 * np.exp(-((t - t0) / 3e7) ** 2) * np.cos(3e-8 * (t - t0))

    def hx(t):
        return 2e-7 * np.exp(-((t - t0) / 3e7) ** 2) * np.sin(3e-8 * (t - t0))

    for quad in (False, True):
        b._det = None
        b.add_burst(0.7, 2.1, hp, hx, psi=0.3, tref=100.0, remove_quad=quad)
        got = {}
        monkeypatch.setattr(deterministic, "_inject", lambda psr, name, params, seconds: got.update({psr.name: seconds}))
        for i, p in enumerate(psrs):
            deterministic.add_burst(p, 0.7, 2.1, hp, hx, psi=0.3, tref=100.0, remove_quad=quad)
            assert np.array_equal(b._det[i], got[p.name][b.order[i]])
        monkeypatch.undo()


def test_kernels_have_no_spills_or_stack():
    from __graft_entry__ import CSRC, NVCC_FLAGS, _nvcc
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_nvcc()] + NVCC_FLAGS + ["-Xptxas", "-v", "-o", os.path.join(d, "lib.so"),
                                                   os.path.join(CSRC, "ptar.cu")], cwd=d, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    found = 0
    for name in ("burst_ninv_kernel", "burst_project_kernel", "burst_reduce_kernel", "burst_psr_kernel"):
        m = re.search(name + r"[^\n]*'[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", text)
        assert m, name
        assert m.groups() == ("0", "0", "0"), (name, m.groups())
        found += 1
    assert found == 4
