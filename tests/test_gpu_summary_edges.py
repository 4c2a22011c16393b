"""GPU tests of the summary kernels -- curn_reduce (run on the CURN and the HD map), fp_reduce + fp_q_int, fe_combine,
the maxima of fe_sky and os_aniso_reduce, os_null_count -- fed constructed inputs through the C ABI and held to the
extended-precision reference of tests/summary_reference.py: both priors, non-uniform grids, every upper-limit quantile,
ties placed across threads / strides / tree halves, exp underflow and flat CDFs, every branch of Q(P, x), and the one
rule for non-finite inputs (include/ptar.h).  Data edge cases only: every launch is an ordinary, in-bounds one."""
import ctypes as C

import numpy as np
import pytest

from tests import reduction_reference as RR
from tests import summary_reference as SR

pytestmark = pytest.mark.gpu

REPORT = RR.Report()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[summary] per kernel family:\n  " + "\n  ".join(REPORT.lines()))


def _t(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _empty(shape, dtype="float64"):
    import torch
    return torch.full(shape if isinstance(shape, tuple) else (shape,), -7, dtype=getattr(torch, dtype), device="cuda")


def _run(fn, *args):
    import torch
    from pta_replicator_b200 import _cabi
    _cabi.check(fn(*args, _cabi.current_stream()), fn.__name__)
    torch.cuda.synchronize()


# ------------------------------------------------------------------ ptar_curn_reduce
def curn_reduce(st, ul, maps):
    """ptar_curn_reduce on ``maps`` [R, NG, NA] with a hand-built model: only the grid fields are read."""
    from pta_replicator_b200 import _cabi
    R, NG, NA = maps.shape
    dev = {k: _t(st[k]) for k in ("log10_A", "wg", "wx", "prior")}
    m = _cabi.CurnModel(n_gamma=NG, n_amp=NA, log10_A=dev["log10_A"].data_ptr(), wg=dev["wg"].data_ptr(),
                        wx=dev["wx"].data_ptr(), prior=dev["prior"].data_ptr(), ul=float(ul))
    lnL = _t(maps)
    out = dict(lnL_max=_empty(R), ml_gamma_index=_empty(R, "int64"), ml_log10_A_index=_empty(R, "int64"),
               ln_bayes=_empty(R), post_log10_A=_empty((R, NA)), post_gamma=_empty((R, NG)), log10_A_ul=_empty(R))
    _run(_cabi.lib().ptar_curn_reduce, lnL.data_ptr(), R, C.addressof(m), *(out[k].data_ptr() for k in (
        "lnL_max", "ml_gamma_index", "ml_log10_A_index", "ln_bayes", "post_log10_A", "post_gamma", "log10_A_ul")))
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("NA,NG", SR.GRIDS)
@pytest.mark.parametrize("spacing", SR.SPACINGS)
def test_curn_reduce_constructed_maps(NA, NG, spacing):
    x, g = SR.grid(NA, NG, spacing)
    names, maps = SR.curn_maps(x, g)
    worst = 0.0
    for kind in SR.PRIORS:
        st = SR.statics(x, g, kind)
        core = SR.curn_core(maps, x, g, st["wg"], st["wx"], st["prior"])
        last = None
        for ul in SR.ULS:
            ref = {k: v for k, v in core.items() if not k.startswith("_")}
            ref["log10_A_ul"] = SR.curn_ul(core, ul)
            got = curn_reduce(st, ul, maps)
            worst = max(worst, SR.curn_compare(got, ref, f"{NA}x{NG} {spacing} {kind} ul={ul}", REPORT, "curn_reduce"))
            q = got["log10_A_ul"]
            assert np.all((q >= x[0]) & (q <= x[-1])), "the upper limit left the grid"
            assert last is None or np.all(q >= last), "the upper limit decreased with the quantile"
            last = q
            assert np.all(np.isfinite(got["post_log10_A"])) and np.all(got["post_log10_A"] >= 0)
    print(f"\n[summary] curn_reduce {NA}x{NG} {spacing}, {len(names)} maps x 2 priors x 4 ul: worst |d|/bound {worst:.3f}")


def test_curn_reduce_is_independent_of_realization_index_and_nreal():
    x, g = SR.grid(97, 57, "geometric")
    names, maps = SR.curn_maps(x, g)
    st = SR.statics(x, g, "uniform")
    one = curn_reduce(st, 0.95, maps)
    R = len(maps)
    idx = (np.arange(257) * 7 + 3) % R
    many = curn_reduce(st, 0.95, maps[idx])
    for k, v in one.items():
        assert np.array_equal(many[k], v[idx], equal_nan=True), k
    for j in (0, R // 2, R - 1):
        single = curn_reduce(st, 0.95, maps[j:j + 1])
        for k, v in one.items():
            assert np.array_equal(single[k], v[j:j + 1], equal_nan=True), (k, names[j])


@pytest.mark.parametrize("NA,NG", [(3, 2), (64, 5), (255, 1), (256, 256)])
def test_curn_reduce_non_finite_rule(NA, NG):
    """The first NaN ranks above every number; a NaN or +inf makes every integral NaN -- the upper limit too, never the
    last node; -inf is a zero likelihood; the all -inf map has ln_bayes = -inf at (0, 0)."""
    x, g = SR.grid(NA, NG, "geometric")
    names, maps = SR.curn_nonfinite_maps(x, g)
    st = SR.statics(x, g, "log-uniform")
    ref = SR.curn_summaries(maps, x, g, st["wg"], st["wx"], st["prior"], 0.95)
    got = curn_reduce(st, 0.95, maps)
    SR.curn_compare(got, ref, f"{NA}x{NG} non-finite", REPORT, "curn_reduce")
    for r, name in enumerate(names):
        if name.startswith(("nan", "inf", "+inf", "two NaN")):
            assert np.isnan(got["log10_A_ul"][r]) and np.isnan(got["ln_bayes"][r]), name
            assert np.all(np.isnan(got["post_log10_A"][r])) and np.all(np.isnan(got["post_gamma"][r])), name
        elif name == "all -inf":
            assert got["lnL_max"][r] == -np.inf and got["ln_bayes"][r] == -np.inf and np.isnan(got["log10_A_ul"][r])
            assert got["ml_gamma_index"][r] == 0 and got["ml_log10_A_index"][r] == 0
        else:
            assert np.isfinite(got["log10_A_ul"][r]) and np.isfinite(got["ln_bayes"][r]), name


# ------------------------------------------------------------------ ptar_fp_reduce_fap
def fp_reduce(amps, fap=True):
    from pta_replicator_b200 import _cabi
    R, P, nc = amps.shape
    nf = nc // 2
    dummy = _t(np.zeros(4))
    m = _cabi.FpModel(n_psr=P, n_freq=nf, n_cb=(2 * nf + 63) // 64, ld=4, Ct=dummy.data_ptr(), psr_order=dummy.data_ptr(),
                      seg_off=dummy.data_ptr(), seg_len=dummy.data_ptr())
    a = _t(amps)
    out = dict(Fp=_empty((R, nf)), Fp_max=_empty(R), Fp_argmax=_empty(R, "int64"), fap=_empty((R, nf)))
    _run(_cabi.lib().ptar_fp_reduce_fap, a.data_ptr(), R, C.addressof(m), out["Fp"].data_ptr(), out["Fp_max"].data_ptr(),
         out["Fp_argmax"].data_ptr(), out["fap"].data_ptr() if fap else None)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check_fp(got, amps, P, tag, exact=None):
    ref = SR.fp_summaries(amps, P)
    SR.check(got["Fp"], ref["Fp"], f"{tag} Fp", REPORT, "fp_reduce")
    if exact is not None:
        assert np.array_equal(got["Fp"], exact, equal_nan=True), f"{tag}: Fp is not the constructed value"
    am = np.array([SR.first_max(row) for row in got["Fp"]])
    assert np.array_equal(got["Fp_argmax"], am), f"{tag}: argmax {got['Fp_argmax']} != {am}"
    assert np.array_equal(got["Fp_max"], got["Fp"][np.arange(len(am)), am], equal_nan=True)
    q, qb = SR.q_ref(P, got["Fp"])                                           # fap is a function of the fp64 Fp
    SR.check(got["fap"], SR._out(q, qb), f"{tag} fap", REPORT, "fp_q_int")


@pytest.mark.parametrize("P", (1, 2, 15, 16, 17, 67, 128))
@pytest.mark.parametrize("Nf", (1, 2, 255, 256))
def test_fp_reduce_fap_constructed_values(P, Nf):
    xs = SR.fp_x_values(P)
    amps = SR.fp_amps_of(xs, P, Nf)
    want = xs[(np.arange(len(xs))[:, None] + np.arange(Nf)[None, :]) % len(xs)]
    got = fp_reduce(amps)
    _check_fp(got, amps, P, f"P={P} Nf={Nf}", exact=want)
    assert np.all(got["fap"][want == 0] == 1.0) and np.all(got["fap"][np.isinf(want)] == 0.0)
    _check_fp(fp_reduce(SR.fp_amps_of(xs[:-1], P, Nf, split=True)), SR.fp_amps_of(xs[:-1], P, Nf, split=True), P,
              f"P={P} Nf={Nf} split")


@pytest.mark.parametrize("Nf", (2, 255, 256))
def test_fp_reduce_ties_and_non_finite(Nf):
    """Equal maxima at f and f + 128, f and f + 1, everywhere; NaN / +inf first, last, at 128 and in the middle: the
    first NaN wins wherever it sits, otherwise the first maximum; fap of a NaN Fp is NaN."""
    P = 3
    rows = []
    base = np.linspace(1.0, 2.0, Nf)
    for a, c in ((5, 133), (133, 134), (0, Nf - 1), (127, 128), (Nf - 2, Nf - 1)):
        if max(a, c) < Nf and a != c:
            v = base.copy()
            v[[a, c]] = 8.0
            rows.append(v)
    rows.append(np.full(Nf, 2.0))
    for val in (np.nan, np.inf):
        for p in SR.positions(Nf):
            v = base.copy()
            v[p] = val
            rows.append(v)
    pos = SR.positions(Nf)
    v = base.copy()
    v[pos[0]], v[pos[-1]] = np.inf, np.nan
    rows.append(v)
    v = base.copy()
    v[pos[-1]] = v[pos[1]] = np.nan
    rows.append(v)
    want = np.stack(rows)
    amps = np.zeros((len(rows), P, 2 * Nf))
    for r in range(len(rows)):
        for f in range(Nf):
            x = want[r, f]
            amps[r, (r + f) % P, 2 * f:2 * f + 2] = (np.nan, 0.0) if np.isnan(x) else SR.exact_pair(x)
    got = fp_reduce(amps)
    _check_fp(got, amps, P, f"ties Nf={Nf}", exact=want)
    assert np.array_equal(np.isnan(got["fap"]), np.isnan(want))
    nan_rows = np.isnan(want).any(axis=1)
    assert np.all(np.isnan(got["Fp_max"][nan_rows])) and np.all(np.isfinite(got["Fp_max"][~nan_rows]) | np.isinf(got["Fp_max"][~nan_rows]))
    assert np.array_equal(got["Fp_argmax"][nan_rows], np.argmax(np.isnan(want[nan_rows]), axis=1))
    no_fap = fp_reduce(amps, fap=False)
    assert np.array_equal(no_fap["Fp_argmax"], got["Fp_argmax"]) and np.all(no_fap["fap"] == -7)


# ------------------------------------------------------------------ ptar_fe_combine
def _maxima_rows(n, rng):
    """Rows of length n: noise, ties, all equal, and NaN / +inf / -inf at ``SR.positions``."""
    base = rng.standard_normal(n)
    rows = [base.copy(), np.full(n, 3.0), np.full(n, -np.inf)]
    for a, c in ((5, 261), (3, 200), (0, n - 1), (127, 128), (n - 2, n - 1), (130, 263)):
        if 0 <= min(a, c) and max(a, c) < n and a != c:
            v = base.copy()
            v[[a, c]] = 9.0
            rows.append(v)
    for val in SR.NONFINITE:
        for p in SR.positions(n):
            v = base.copy()
            v[p] = val
            rows.append(v)
    pos = SR.positions(n)
    if len(pos) > 1:
        v = base.copy()
        v[pos[0]], v[pos[-1]] = np.inf, np.nan
        rows.append(v)
        v = base.copy()
        v[pos[-1]] = v[pos[1]] = np.nan
        rows.append(v)
    return np.stack(rows)


@pytest.mark.parametrize("Nf", (1, 2, 255, 256))
@pytest.mark.parametrize("R", (1, 255, 257))
def test_fe_combine_direct(Nf, R):
    from pta_replicator_b200 import _cabi
    rng = np.random.default_rng(Nf + R)
    pool = _maxima_rows(Nf, rng)
    fmax = pool[(np.arange(R) * 5 + 1) % len(pool)]
    farg = rng.integers(0, 12288, (R, Nf))
    dummy = _t(np.zeros(4))
    m = _cabi.FeModel(n_psr=1, n_freq=Nf, n_sky=1, n_sb=1, kp=16, Lf=dummy.data_ptr(), ant=dummy.data_ptr(), linv=dummy.data_ptr())
    a, b = _t(fmax), _t(farg)
    out = dict(fe_max=_empty(R), argmax_f=_empty(R, "int64"), argmax_sky=_empty(R, "int64"))
    _run(_cabi.lib().ptar_fe_combine, a.data_ptr(), b.data_ptr(), R, C.addressof(m), *(v.data_ptr() for v in out.values()))
    ref = SR.fe_combine(fmax, farg)
    for k, v in out.items():
        assert np.array_equal(v.cpu().numpy(), ref[k], equal_nan=True), k


# ------------------------------------------------------------------ os_aniso_reduce and os_null_count, fed directly
def _os_stub():
    """A minimal valid ptar_os_model (2 pulsars, one pair) for the stage-3 entry points, which read none of it."""
    from pta_replicator_b200 import _cabi
    d = _t(np.zeros(64))
    return _cabi.OsModel(n_psr=2, n_tiles=0, nc=2, ncp=8, sqrt_phi=d.data_ptr(), n_pairs=1, n_orf=1, pairs=d.data_ptr()), d


@pytest.mark.parametrize("n_sky", (1, 2, 255, 256, 257, 600))
def test_os_aniso_reduce_direct(n_sky):
    """Stage 3 of ptar_os_aniso on a given radiometer row: ties in one thread's stride (k, k + 256), across threads and
    tree halves go to the lower pixel; the first NaN ranks above every number; the map is copied bit for bit."""
    from pta_replicator_b200 import _cabi
    rows = _maxima_rows(n_sky, np.random.default_rng(n_sky))
    R = len(rows)
    osm, d = _os_stub()
    am = _cabi.OsAnisoModel(n_lm=0, n_z=0, n_sky=n_sky, n_col=n_sky, n_colp=(n_sky + 63) // 64 * 64, kd=1, kdp=32,
                            V=d.data_ptr(), dsqrt=d.data_ptr())
    mp = _t(rows)
    out = dict(snr_max=_empty(R), argmax=_empty(R, "int64"), radio=_empty((R, n_sky)))
    _run(_cabi.lib().ptar_os_aniso_stage, d.data_ptr(), R, C.addressof(osm), C.addressof(am), d.data_ptr(), mp.data_ptr(),
         None, None, None, out["snr_max"].data_ptr(), out["argmax"].data_ptr(), out["radio"].data_ptr(), 3)
    am_ref = np.array([SR.first_max(r) for r in rows])
    assert np.array_equal(out["argmax"].cpu().numpy(), am_ref)
    assert np.array_equal(out["snr_max"].cpu().numpy(), rows[np.arange(R), am_ref], equal_nan=True)
    assert np.array_equal(out["radio"].cpu().numpy(), rows, equal_nan=True)


@pytest.mark.parametrize("n_col", (2, 3, 256, 257, 258, 1000))
def test_os_null_count_direct(n_col):
    """Stage 3 of ptar_os_null on given S/N rows: exceedances count ties and NaN null columns; the p-value of a NaN
    observed S/N is NaN."""
    from pta_replicator_b200 import _cabi
    rng = np.random.default_rng(n_col)
    base = rng.standard_normal(n_col)
    rows = [base.copy(), np.zeros(n_col), np.full(n_col, np.inf)]
    for val in SR.NONFINITE:
        for p in SR.positions(n_col):
            v = base.copy()
            v[p] = val
            rows.append(v)
    v = base.copy()
    v[1:] = np.nan
    rows.append(v)
    v = base.copy()
    v[n_col // 2:] = base[0]
    rows.append(v)
    snr = np.stack(rows)
    R = len(snr)
    osm, d = _os_stub()
    nl = _cabi.OsNullModel(method=_cabi.OS_NULL_SKY_SCRAMBLE, n_col=n_col, n_colp=(n_col + 63) // 64 * 64, kd=1, kdp=32,
                           V=d.data_ptr(), dsqrt=d.data_ptr())
    s = _t(snr)
    ex, fap = _empty(R, "int64"), _empty(R)
    _run(_cabi.lib().ptar_os_null_stage, d.data_ptr(), R, C.addressof(osm), C.addressof(nl), d.data_ptr(), s.data_ptr(),
         ex.data_ptr(), fap.data_ptr(), 3)
    ref = SR.null_count(snr)
    assert np.array_equal(ex.cpu().numpy(), ref["null_exceed"])
    assert np.array_equal(fap.cpu().numpy(), ref["fap"], equal_nan=True)
    assert np.isnan(fap.cpu().numpy()[3]) and not np.isnan(ref["fap"][0])     # row 3: NaN observed S/N


# ------------------------------------------------------------------ repeated sky directions through a batch
def _rows(b, R, seed):
    rng = np.random.default_rng(seed)
    rows = np.zeros((R, b.ld))
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        rows[:, s:s + n] = rng.standard_normal((R, n)) * b.err_s[i]
    return rows


def _repeated_sky(n_dir, reps, seed=5):
    """[n_dir * reps, 2]: direction i % n_dir at index i, so every value of a map is an n-fold tie."""
    rng = np.random.default_rng(seed)
    d = np.stack([np.arccos(rng.uniform(-0.9, 0.9, n_dir)), rng.uniform(0, 2 * np.pi, n_dir)], axis=1)
    return np.tile(d, (reps, 1))


def test_fe_sky_repeated_directions():
    """21 directions listed 4 times (indices i, i + 21, i + 42, i + 63: different stages, quads and column halves of
    fe_sky): the copies are bit-equal in the map and every maximum reports the lowest index."""
    b = RR.edge_batch((64, 65, 193, 70, 80), seed=3)
    b.set_fp_statistic(n_freqs=5)
    b.set_fe_statistic(sky=_repeated_sky(21, 4))
    res = b.fp_statistic_of(_t(_rows(b, 40, 1)), maps=True)
    fe = res["Fe"].cpu().numpy()                                             # [R, Nf, 84]
    assert np.array_equal(fe[..., :21], fe[..., 21:42]) and np.array_equal(fe[..., :21], fe[..., 63:])
    arg = res["Fe_fargmax"].cpu().numpy()
    assert np.array_equal(arg, np.argmax(fe, axis=2)) and arg.max() < 21
    assert np.array_equal(res["Fe_argmax_sky"].cpu().numpy(), arg[np.arange(40), res["Fe_argmax_f"].cpu().numpy()])


def test_radiometer_repeated_directions():
    """21 directions listed 25 times (525 pixels: every thread of os_aniso_reduce strides, the copies sit in different
    threads): copies with bit-equal statics are bit-equal in the map and the lowest pixel is reported."""
    b = RR.edge_batch((64, 65, 193, 70, 80), seed=4)
    b.set_optimal_statistic(components=5, orfs=("hd",))
    b.set_os_anisotropy(sky=_repeated_sky(21, 25))
    res = b.optimal_statistic_of(_t(_rows(b, 40, 2)), aniso_maps=True)
    mp = res["radio_snr"].cpu().numpy()
    an = b.compile()["os"]["aniso"]
    V = an["dev"]["V"].cpu().numpy().reshape(an["model"].n_colp, an["model"].kdp)[:525]
    ds = an["dev"]["dsqrt"].cpu().numpy()[:525]
    # a copy whose host statics are bit-equal to the first listing's (numpy may round a trailing column differently)
    same = np.array([np.array_equal(V[c], V[c % 21]) and ds[c] == ds[c % 21] for c in range(525)])
    assert same.sum() >= 400
    assert np.array_equal(mp[:, same], mp[:, np.arange(525)[same] % 21])
    arg = res["radio_argmax"].cpu().numpy()
    assert np.array_equal(arg, np.argmax(mp, axis=1)) and np.all(same[:42]) and np.all(arg[same[arg]] < 21)
    assert np.array_equal(res["radio_snr_max"].cpu().numpy(), mp[np.arange(40), arg])
