"""GPU edge sweep of the per-realization reductions -- timing fit, optimal statistic, its null distributions and the
Fp-statistic -- against the extended-precision reference of tests/reduction_reference.py, every output within its
rigorous componentwise bound.  The shapes sit at the kernels' edges (see the table in that module and the coverage test
of tests/test_reduction_edges_cpu.py): pulsars whose only chunk is partial, ring wraps, tile splits, every os_project
and timing instantiation, partial and full column blocks, R across the realization-block edges.  Also: poisoned
alignment slots and ld tails change nothing, the timing fit leaves padding untouched, staged launches equal fused
ones, and the Fp false-alarm probability is Q(P, Fp) to 1e-12."""
import numpy as np
import pytest

from tests import reduction_reference as RR

pytestmark = pytest.mark.gpu

REPORT = RR.Report()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[edges] per kernel family:\n  " + "\n  ".join(REPORT.lines()))


def _rows(b, R, seed, f0=None, models=True):
    """[R, ld] fp64 rows, zero padded: r % 4 == 0 noise (the TOA uncertainties), 1 all zero, 2 almost in the pulsar's
    quadratic span (1e-5 s model, 1e-11 s off it), 3 a sinusoid at f0 (default 7 / span) plus noise."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((R, b.ld))
    for i in range(b.n_psr):
        s, n, t = b.toa_off[i], b.ntoa[i], b.t_tdb[i]
        x = (t - t.mean()) / max(np.ptp(t), 1.0)
        f = 7.0 / max(np.ptp(np.concatenate(b.t_tdb)), 1.0) if f0 is None else f0
        for r in range(R):
            k = r % 4
            if k == 0:
                rows[r, s:s + n] = rng.standard_normal(n) * b.err_s[i]
            elif k == 2:
                rows[r, s:s + n] = 1e-5 * (rng.standard_normal(3) @ np.stack([np.ones(n), x, x * x])) + 1e-11 * rng.standard_normal(n)
            elif k == 3:
                rows[r, s:s + n] = 2e-5 * np.sin(2 * np.pi * f * t + 0.3 * i) + rng.standard_normal(n) * b.err_s[i]
    return rows


def _poison(b, rows):
    """The rows with every alignment slot and the ld tail set to NaN, +inf, -inf (cycling)."""
    p = rows.copy()
    vals = np.array([np.nan, np.inf, -np.inf])
    pad = np.ones(b.ld, dtype=bool)
    for s, n in zip(b.toa_off, b.ntoa):
        pad[s:s + n] = False
    idx = np.flatnonzero(pad)
    p[:, idx] = vals[np.arange(idx.size) % 3][None, :]
    return p, idx


def _t(b, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(b.device)


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items() if hasattr(v, "cpu")}


def _equal(a, c, keys):
    import torch
    for k in keys:
        assert torch.equal(a[k], c[k]), k


# ------------------------------------------------------------------ optimal statistic
def _os_statics(b):
    st = b.compile()["os"]
    m = st["model"]
    g = {k: st[k].cpu().numpy() for k in ("C", "sqrt_phi", "pairs", "t_ab", "orf", "dnorm", "dsqrt", "finv")}
    g.update(nc=m.nc, seg_off=np.asarray(b.toa_off), seg_len=np.asarray(b.ntoa))
    g["C"] = g["C"].reshape(b.ld, m.ncp)
    g["orf"] = g["orf"].reshape(m.n_orf, m.n_pairs)
    g["finv"] = g["finv"].reshape(m.n_orf, m.n_orf)
    return g


def _check_os(b, rows, res, tag):
    ref = RR.optimal_statistic(_os_statics(b), rows)
    for k in ("rho", "A2", "snr", "A2_mc"):
        RR.check(res[k].cpu().numpy(), ref[k], f"{tag} {k}", REPORT, "os_" + ("pairs" if k != "rho" else "rho"))
    return ref


@pytest.fixture(scope="module")
def edge():
    return RR.edge_batch(RR.EDGE_NTOAS, seed=11)


@pytest.mark.parametrize("K,kind,R", RR.os_cases() + [(16, "all4", 1025)])
def test_optimal_statistic_edges(edge, K, kind, R):
    b = edge
    b.set_optimal_statistic(components=K, orfs=RR.templates(b.n_psr, kind))
    rows = _rows(b, R, seed=K)
    res = b.optimal_statistic_of(_t(b, rows), pairs=True)
    _check_os(b, rows, res, f"K={K} {kind} R={R}")
    keys = ("rho", "A2", "snr", "A2_mc")
    if R <= 130:
        pois, _ = _poison(b, rows)
        _equal(res, b.optimal_statistic_of(_t(b, pois), pairs=True), keys)
        _equal(res, b.optimal_statistic_of(_t(b, rows), pairs=True, timers={}), keys)
    assert np.all(res["rho"].cpu().numpy()[1::4] == 0.0)          # all-zero rows


@pytest.mark.parametrize("npsr", [2, 256])
def test_optimal_statistic_pulsar_count_limits(npsr):
    """2 pulsars (one pair, 255 idle threads in the pair tree) and the 256-pulsar limit (32,640 pairs, 72 KB of shared
    memory) with four templates including a user matrix (one pair admits only one template)."""
    rng = np.random.default_rng(npsr)
    ntoas = (5, 65) if npsr == 2 else tuple(int(n) for n in rng.integers(8, 41, npsr))
    b = RR.edge_batch(ntoas, seed=npsr, tm_min=24)
    b.set_optimal_statistic(components=5, orfs=RR.templates(b.n_psr, "hd" if npsr == 2 else "all4"))   # one pair: one template
    R = 65 if npsr == 2 else 3
    rows = _rows(b, R, seed=npsr)
    res = b.optimal_statistic_of(_t(b, rows), pairs=True)
    _check_os(b, rows, res, f"P={npsr}")
    pois, _ = _poison(b, rows)
    _equal(res, b.optimal_statistic_of(_t(b, pois), pairs=True), ("rho", "A2", "snr", "A2_mc"))


# ------------------------------------------------------------------ null distributions
@pytest.mark.parametrize("method,n,K,P,R", RR.null_cases())
def test_os_null_edges(method, n, K, P, R):
    b = RR.edge_batch(RR.null_ntoas(P), seed=100 + P + K)
    b.set_optimal_statistic(components=K, orfs=("hd",))
    b.set_os_null(method, n=n, seed=n, match=None if P <= 3 else 0.5)
    rows = _rows(b, R, seed=n + K)
    res = b.optimal_statistic_of(_t(b, rows), null_values=True)
    st = b.compile()["os"]["null"]
    nm = st["model"]
    N = dict(method=method, V=st["dev"]["V"].cpu().numpy().reshape(nm.n_colp, nm.kdp), kd=nm.kd, n_col=nm.n_col,
             dsqrt=st["dev"]["dsqrt"].cpu().numpy())
    ref = RR.os_null(_os_statics(b), N, RR.optimal_statistic(_os_statics(b), rows))
    ns = res["null_snr"].cpu().numpy()
    RR.check(ns, ref["snr"], f"{method} n={n} K={K} P={P} R={R} null S/N", REPORT, "os_null")
    ex = res["null_exceed"].cpu().numpy()
    assert np.all(ref["exceed_lo"] <= ex) and np.all(ex <= ref["exceed_hi"])
    assert np.array_equal(ex, np.sum(ns[:, 1:] >= ns[:, :1], axis=1))
    assert np.array_equal(res["fap"].cpu().numpy(), (1.0 + ex) / (n + 1))
    keys = ("null_snr", "null_exceed", "fap", "snr")
    pois, _ = _poison(b, rows)
    _equal(res, b.optimal_statistic_of(_t(b, pois), null_values=True), keys)
    _equal(res, b.optimal_statistic_of(_t(b, rows), null_values=True, timers={}), keys)


# ------------------------------------------------------------------ Fp-statistic
def _fp_check(b, rows, res, tag):
    from pta_replicator_b200.engine import fp_whitened_basis
    st = b.compile()["fp"]
    pf = dict(Ct=st["Ct"].cpu().numpy(), n_freq=st["n_freq"])
    Ct = [fp_whitened_basis(pf, s, n) for s, n in zip(b.toa_off, b.ntoa)]
    ref = RR.fp_statistic(Ct, b.toa_off, b.ntoa, rows)
    R, Nf = rows.shape[0], st["n_freq"]
    RR.check(res["amps"].cpu().numpy().reshape(R, b.n_psr, 2 * Nf), ref["amps"], f"{tag} amps", REPORT, "fp_project")
    Fp = res["Fp"].cpu().numpy()
    RR.check(Fp, ref["Fp"], f"{tag} Fp", REPORT, "fp_reduce")
    # max / argmax wherever the top two reference values are farther apart than their bounds
    fh, fb = ref["Fp"]["hi"], ref["Fp"]["bound"]
    o = np.argsort(-fh, axis=1, kind="stable")
    r = np.arange(R)
    if Nf > 1:
        sep = fh[r, o[:, 0]] - fh[r, o[:, 1]] > fb[r, o[:, 0]] + fb[r, o[:, 1]]
    else:
        sep = np.ones(R, dtype=bool)
    am = res["Fp_argmax"].cpu().numpy()
    assert np.array_equal(am[sep], o[sep, 0]), tag
    assert np.array_equal(res["Fp_max"].cpu().numpy(), Fp[r, am])
    return ref


def _fap_check(P, Fp, fap, tag):
    q = RR.q_int(P, Fp.ravel(), np.longdouble).astype(float).reshape(Fp.shape)
    keep = q >= 1e-300
    rel = float(np.max(np.abs(fap[keep] - q[keep]) / q[keep])) if keep.any() else 0.0
    REPORT.add("fp_fap", rel / 1e-12, rel / RR.U)
    print(f"\n[fp] {tag}: FAP worst relative error {rel:.1e} against Q(P, Fp) over {int(keep.sum())} values, "
          f"Fp in [{Fp.min():.2f}, {Fp.max():.2f}]")
    assert rel <= 1e-12, tag
    assert np.all(fap[~keep] <= 1e-290)


@pytest.mark.parametrize("nf,R", RR.fp_cases())
def test_fp_statistic_edges(edge, nf, R):
    b = edge
    T = max(np.ptp(np.concatenate(b.t_tdb)), 1.0)
    if nf == "unsorted":
        freqs = np.random.default_rng(5).permutation(np.r_[np.arange(1, 20), 7.5]) / T
        b.set_fp_statistic(freqs=freqs)
        f0 = 7.0 / T
    else:
        b.set_fp_statistic(n_freqs=nf)
        f0 = min(7, nf) / T
    freqs = b._fp["freqs"]
    rows = _rows(b, R, seed=3 + R, f0=f0)
    res = b.fp_statistic_of(_t(b, rows), pulsars=True)
    _fp_check(b, rows, res, f"Nf={nf} R={R}")
    Fp, fap = res["Fp"].cpu().numpy(), res["fap"].cpu().numpy()
    _fap_check(b.n_psr, Fp, fap, f"Nf={nf} R={R}")
    z = np.arange(R) % 4 == 1
    assert np.all(Fp[z] == 0.0) and np.all(res["Fp_argmax"].cpu().numpy()[z] == 0) and np.all(fap[z] == 1.0)
    planted = np.arange(R) % 4 == 3
    if planted.any():
        assert np.all(res["Fp_argmax"].cpu().numpy()[planted] == int(np.argmin(np.abs(freqs - f0))))
    keys = ("Fp", "Fp_max", "Fp_argmax", "fap", "amps")
    pois, _ = _poison(b, rows)
    _equal(res, b.fp_statistic_of(_t(b, pois), pulsars=True), keys)
    _equal(res, b.fp_statistic_of(_t(b, rows), pulsars=True, timers={}), keys)


@pytest.mark.parametrize("P", [2, 24, 67, 256])
def test_fp_fap_matches_q_on_null_rows(P):
    """Rows from the batch's own noise model: Fp ~ Gamma(P, 1), so the FAP is exercised where Fp ~ P."""
    rng = np.random.default_rng(P)
    ntoas = tuple(int(n) for n in rng.integers(8, 41, P)) if P > 24 else RR.null_ntoas(P)
    b = RR.edge_batch(ntoas, seed=200 + P, tm_min=24)
    b.set_fp_statistic(n_freqs=20)
    res = b.fp_statistic(130, seed=P)
    _fap_check(P, res["Fp"].cpu().numpy(), res["fap"].cpu().numpy(), f"null rows P={P}")


# ------------------------------------------------------------------ timing fit
def _timing_run(b, rows_t, R, stage=None):
    from pta_replicator_b200 import _cabi
    L = _cabi.lib()
    keep = []
    tmx = b._timing_job(b.compile(), R, keep)
    out = rows_t.clone()
    s = _cabi.current_stream()
    if stage is None:
        _cabi.check(L.ptar_timing_project(out.data_ptr(), b.ld, R, *tmx, s), "ptar_timing_project")
    else:
        for k in (1, 2):
            _cabi.check(L.ptar_timing_project_stage(out.data_ptr(), b.ld, R, *tmx, k, s), "ptar_timing_project")
    return out


@pytest.mark.parametrize("kmax,R", list(zip(RR.TM_KMAX, (1, 15, 16, 17, 31, 32, 33, 100))))
def test_timing_fit_edges(kmax, R):
    """Mixed k in one batch, pulsars without a model, every column bucket; padding untouched."""
    ntoas = (5, 6, 7, 40, 64, 65, 193, 1025, 2100)
    b = RR.edge_batch(ntoas, seed=300 + kmax, tm=False)
    ks = []
    for i, n in enumerate(ntoas):
        n_ep = np.unique(np.round(b.t_tdb[i] / 10.0)).size       # sub-band TOAs of an epoch share every smooth column
        k = 0 if i == 1 else min(kmax if i == len(ntoas) - 1 else 1 + (i * 7) % kmax, n_ep - 1)
        if k:
            poly, extra = RR.tm_columns(b, i, k)
            b.set_timing_model(i, poly=poly, extra=extra)
        ks.append(k)
    assert max(ks) == kmax
    rows = _rows(b, R, seed=kmax)
    st = b.compile()["tm"]
    T = {k: st[k].cpu().numpy() for k in ("k", "q_off", "Q", "sqrtw", "seg_off", "seg_len")}
    got = _timing_run(b, _t(b, rows), R).cpu().numpy()
    RR.check(got, RR.timing_fit(T, rows), f"kmax={kmax} R={R}", REPORT, "timing")
    fitted = np.zeros(b.ld, dtype=bool)
    for s, n, k in zip(b.toa_off, ntoas, ks):
        fitted[s:s + n] = k > 0
    assert np.array_equal(got[:, ~fitted], rows[:, ~fitted])          # no model, alignment slots, ld tail: untouched
    pois, idx = _poison(b, rows)
    gp = _timing_run(b, _t(b, pois), R).cpu().numpy()
    real = np.setdiff1d(np.arange(b.ld), idx)
    assert np.array_equal(gp[:, real], got[:, real])
    assert np.array_equal(gp[:, idx], pois[:, idx], equal_nan=True)     # the padding still holds the poison
    assert np.array_equal(_timing_run(b, _t(b, rows), R, stage=True).cpu().numpy(), got)
