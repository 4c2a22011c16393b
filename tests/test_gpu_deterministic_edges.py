"""GPU edge sweep of the Fourier-basis, Cholesky, CW, CW-catalog, burst and memory kernels -- ptar_fourier_basis (Ftile
from compile() and create_fourier_design_matrix_red), ptar_cholesky_lower, ptar_cgw_delay (through PulsarBatch.add_cgw),
ptar_cw_catalog (prefactors, sources x TOAs, slice reduction), ptar_burst_delay and ptar_memory_delay -- against the
extended-precision reference of tests/deterministic_reference.py, every output within its componentwise bound (burst
and memory bit-exact).  Also: rows past a tile's epoch count and alignment slots are exactly 0, the strict upper
triangle of L is 0, info names the first leading minor that is not positive definite, batched factors equal single
ones bit for bit, catalog calls are repeatable bit for bit, and guards past every output and scratch stay untouched."""
import ctypes as C

import numpy as np
import pytest

from tests import deterministic_reference as DR
from tests import generator_reference as GR
from tests.reduction_reference import EDGE_NTOAS

pytestmark = pytest.mark.gpu

REPORT = DR.Report()
GUARD = 64
SENTINEL = -1.2345678901234567e300


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[deterministic edges] per kernel family:\n  " + "\n  ".join(REPORT.lines()))


def _np(t):
    return t.detach().cpu().numpy()


def _dev(a):
    import torch
    from pta_replicator_b200 import _cabi
    return torch.from_numpy(np.ascontiguousarray(a)).to(_cabi.require_cuda())


def _guarded(n, fill=None):
    """A device buffer of n + GUARD doubles: ``fill`` (or SENTINEL) in the first n, SENTINEL after."""
    a = np.full(n + GUARD, SENTINEL)
    if fill is not None:
        a[:n] = fill
    return _dev(a)


def _guards_ok(buf, n):
    return bool(np.all(_np(buf)[n:] == SENTINEL))


# ------------------------------------------------------------------ Fourier basis
@pytest.mark.parametrize("K", DR.FOURIER_K)
def test_ftile_from_compile(K):
    cases = [("gen", 0), ("gen", 1)] + ([("own", 0), ("own", 1)] if K in (2, 30) else [])
    for kind, conv in cases:
        b = DR.fourier_batch(kind, K, conv)
        st = b.compile()
        ref = DR.ftile(b.plan(), b.t0_table, conv)
        w, _ = DR.check(_np(st["Ftile"]), ref, f"Ftile {kind} K={K} conv={conv}", REPORT, "fourier")
        print(f"Ftile {kind} K={K} conv={conv}: worst |d|/bound {w:.3f}")


def test_design_matrix_phase_path():
    from pta_replicator_b200.red_noise import create_fourier_design_matrix_red
    rng = np.random.default_rng(4)
    worst = 0.0
    for N in (1, 255, 256, 257):
        t = np.sort(rng.uniform(53000, 58800, N)) * 86400.0
        for conv in (False, True):
            for nm in (30, 7):                       # N nm crosses a 256-thread block mid-row
                np.random.seed(100 + N)
                F, ff = create_fourier_design_matrix_red(t, nmodes=nm, Tspan=3e8, pshift=True, libstempo_convention=conv)
                np.random.seed(100 + N)
                ph = np.random.uniform(0.0, 2 * np.pi, nm)
                f = 1.0 * np.arange(1, nm + 1) / 3e8
                assert np.array_equal(ff, np.repeat(f, 2))
                w, _ = DR.check(F, DR.design_matrix(t, f, ph, conv), f"design matrix N={N} conv={conv} nm={nm}", REPORT,
                                "fourier")
                worst = max(worst, w)
    print(f"design matrix (pshift): worst |d|/bound {worst:.3f}")


# ------------------------------------------------------------------ Cholesky
def _chol(As):
    import torch
    from pta_replicator_b200 import _cabi
    A = _dev(np.asarray(As, dtype=np.float64))
    batch, n = A.shape[0], A.shape[1]
    L = torch.full_like(A, SENTINEL)
    info = torch.full((batch,), -7, dtype=torch.int32, device=A.device)
    _cabi.check(_cabi.lib().ptar_cholesky_lower(L.data_ptr(), A.data_ptr(), n, batch, info.data_ptr(),
                                                _cabi.current_stream()), "ptar_cholesky_lower")
    return _np(L), _np(info)


def _check_factor(A, L, what):
    n = A.shape[0]
    assert np.all(np.triu(L, 1) == 0), what
    assert np.all(np.diag(L) > 0), what
    return DR.check(A, DR.cholesky_ref(A, L), what, REPORT, "cholesky")[0]


CHOL_N = (1, 2, 31, 32, 33, 64, 65, 67, 112, 255, 256, 257, 1024)


@pytest.mark.parametrize("n", CHOL_N)
def test_cholesky_within_higham_bound(n):
    rng = np.random.default_rng(n)
    batches = (1, 3, 130) if n <= 67 else ((1, 3) if n <= 257 else (1,))
    kmax = 12 if n <= 257 else 10
    worst = 0.0
    for batch in batches:
        kappas = np.logspace(1, kmax, batch) if batch > 1 else [10.0 ** kmax]
        As = np.stack([DR.spd(n, k, rng) for k in kappas])
        L, info = _chol(As)
        assert np.all(info == 0), info
        for k in range(batch):
            worst = max(worst, _check_factor(As[k], L[k], f"n={n} batch={batch} kappa={kappas[k]:.0e}"))
        if batch > 1 and n <= 67:
            for k in (0, batch // 2, batch - 1):                  # the mixed batch equals one-at-a-time bit for bit
                L1, _ = _chol(As[k:k + 1])
                assert np.array_equal(L1[0], L[k]), (n, batch, k)
    print(f"cholesky n={n}: worst |d|/bound {worst:.3f}")


def test_cholesky_orfs_and_info():
    hd = DR.orf_matrix(DR.ng15_radec("full"))
    an = DR.config4_orf()
    L, info = _chol(np.stack([hd, an]))
    assert np.all(info == 0)
    for A, Lk, what in ((hd, L[0], "HD ng15-full"), (an, L[1], "lmax=6 config4")):
        w = _check_factor(A, Lk, what)
        print(f"cholesky {what}: worst |d|/bound {w:.3f}")
    rng = np.random.default_rng(7)
    n = 64
    As = np.stack([DR.not_pd_at(n, k, rng) for k in (1, 2, 33, n)] + [DR.spd(n, 1e3, rng)])
    _, info = _chol(As)
    assert info.tolist() == [1, 2, 33, n, 0]


# ------------------------------------------------------------------ single CW source through add_cgw
def _cgw_batch(P):
    from pta_replicator_b200.engine import PulsarBatch
    pool = GR.GEN_NTOAS + EDGE_NTOAS
    ntoas = {1: (1025,), 3: (1, (17, 2), 2100)}.get(P) or tuple(pool[j % len(pool)] for j in range(P))
    return PulsarBatch(GR.dense_pulsars(ntoas, seed=P, name="W"))


@pytest.mark.parametrize("P", (1, 3, 67))
def test_cgw_det_through_add_cgw(P):
    b = _cgw_batch(P)
    sel = np.concatenate([np.arange(o, o + n) for o, n in zip(b.toa_off, b.ntoa)])
    pad = np.ones(b.ld, dtype=bool)
    pad[sel] = False
    pdist = np.linspace(0.5, 2.0, P)
    pphase = np.linspace(0.3, 3.0, P)
    sources = DR.CGW_SOURCES + (DR.near_merger(np.concatenate(b.mjd)),)
    worst = {}
    for si, src in enumerate(sources):
        for mode in (0, 1, 2):
            for psr in (0, 1):
                kw = dict(pdist=pdist, pphase=pphase if si % 2 else None, psrTerm=bool(psr), evolve=mode == 0,
                          phase_approx=mode == 1, tref=src[8])
                b._det = None
                b.add_cgw(*src[:8], **kw)
                det = b.plan()["det"]
                assert np.all(det[pad] == 0)
                a = b.cgw_inputs(*src[:8], **kw)
                ref = DR.cgw_ref(a, sel=sel).out()
                assert np.isfinite(ref["hi"]).all()
                w, _ = DR.check(det[sel], ref, f"P={P} source {si} mode {mode} psrTerm {psr}", REPORT, f"cw mode {mode}")
                worst[mode] = max(worst.get(mode, 0.0), w)
    print(f"cgw P={P}: worst |d|/bound per mode " + ", ".join(f"{m}: {w:.3f}" for m, w in sorted(worst.items())))


# ------------------------------------------------------------------ catalog
def _safe_catalog(n_src, seed, t, phat, pdist, pph, use, los):
    """DR.catalog with every source at more than 1e-9 (relative) from a merger at every TOA: offenders get a lower
    fgw until none is left."""
    cat = DR.catalog(n_src, seed=seed, los=los)
    for _ in range(20):
        pre = DR.prefactors_np(cat, phat, pdist, pph, use)
        bad = [s for s in range(n_src) if DR.merger_margin(pre[s:s + 1], t) <= 1e-9]
        if not bad:
            return cat
        cat[4, bad] *= 0.9
    raise AssertionError("could not keep the catalog away from mergers")


@pytest.mark.parametrize("case", DR.CAT_CASES, ids=lambda c: "-".join(map(str, c)))
def test_cw_catalog(case):
    import torch
    from pta_replicator_b200 import _cabi
    n_src, spec, n_toa, tag, acc = case
    ns = DR.n_slices_of(n_src, spec)
    mode, psr, pdist, pph, use = DR.cat_variant(tag)
    rng = np.random.default_rng(n_src * 7 + n_toa)
    los = n_src in (31, 257, 4097)                            # the pulsar at dec +90 deg, source 0 on its line of sight
    ra, dec = rng.uniform(0, 2 * np.pi), (np.pi / 2 if los else np.arcsin(rng.uniform(-1, 1)))
    phat = DR.phat_of(ra, dec)
    t = DR.cat_toas(n_toa, seed=n_src)
    cat = _safe_catalog(n_src, n_src + n_toa, t, phat, pdist, pph, use, los)
    out0 = rng.standard_normal(n_toa) * 1e-7
    t_d, cat_d = _dev(t), _dev(cat)
    out, pre, partial = _guarded(n_toa, out0), _guarded(n_src * 16), _guarded(ns * n_toa)
    ph = (C.c_double * 3)(*phat)

    def run():
        out[:n_toa] = torch.from_numpy(out0).to(out.device)
        _cabi.check(_cabi.lib().ptar_cw_catalog(out.data_ptr(), t_d.data_ptr(), n_toa, ph, cat_d.data_ptr(), n_src, pdist, pph,
                                                use, mode, psr, acc, pre.data_ptr(), partial.data_ptr(), ns,
                                                _cabi.current_stream()), "ptar_cw_catalog")
        return _np(out).copy()

    o1 = run()
    o2 = run()
    assert np.array_equal(o1, o2, equal_nan=True)
    assert _guards_ok(out, n_toa) and _guards_ok(pre, n_src * 16) and _guards_ok(partial, ns * n_toa)
    P = _np(pre)[:n_src * 16].reshape(n_src, 16)
    assert np.all(P[:, 14:] == 0)
    wp, _ = DR.check_nan(P[:, :14], DR.pre_ref(cat, phat, pdist, pph, use), f"pre {case}", REPORT, "cat prefactors")
    if los:
        assert np.isnan(P[0, 10]) and np.isnan(P[0, 11])
    idx = DR.toa_sample(n_toa, n_src, rng)
    ref, rs = DR.catalog_sum_ref(P, t[idx], mode, psr, out0[idx] if acc else None)
    assert np.isfinite(o1[:n_toa]).all()
    ws, _ = DR.check(o1[idx], ref, f"catalog sum {case}", REPORT, "cat sum")
    print(f"catalog {case}: {np.isnan(rs).any(axis=1).sum()} NaN sources, worst |d|/bound pre {wp:.3f}, sum {ws:.3f}")


# ------------------------------------------------------------------ burst and memory
SPECIALS = np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, -2.2250738585072014e-308, np.inf, -np.inf, np.nan, 1.0, -3.5,
                     1e300, -1e-300])


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64))


def _with_specials(x, rng):
    k = min(len(x), len(SPECIALS))
    x[rng.choice(len(x), size=k, replace=False)] = rng.permutation(SPECIALS)[:k]
    return x


@pytest.mark.parametrize("n", (1, 255, 256, 257, 70000))
def test_burst_and_memory_bit_exact(n):
    from pta_replicator_b200 import _cabi
    L, s = _cabi.lib(), _cabi.current_stream()
    rng = np.random.default_rng(n)
    hp = _with_specials(rng.standard_normal(n) * 1e-9, rng)
    hx = _with_specials(rng.standard_normal(n) * 1e-9, rng)
    out0 = _with_specials(rng.standard_normal(n) * 1e-7, rng)
    fplus, fcross, psi = -0.37, 0.81, 0.7
    c2, s2 = float(np.cos(2 * psi)), float(np.sin(2 * psi))
    t0 = 55000.5 * 86400
    t = np.sort(rng.uniform(53000, 58800, n)) * 86400
    t[:: max(1, n // 3)] = t0
    t[1:: max(2, n // 3)] = np.nextafter(t0, -np.inf)
    t = _with_specials(t, rng) if n > 20 else t
    hp_d, hx_d, t_d = _dev(hp), _dev(hx), _dev(t)
    for acc in (0, 1):
        out = _guarded(n, out0)
        _cabi.check(L.ptar_burst_delay(out.data_ptr(), hp_d.data_ptr(), hx_d.data_ptr(), fplus, fcross, c2, s2, acc, n, s))
        rplus = hp * c2 - hx * s2
        rcross = hp * s2 + hx * c2
        with np.errstate(invalid="ignore", over="ignore"):
            res = (-fplus) * rplus - fcross * rcross
        got = _np(out)
        assert _guards_ok(out, n)
        assert _same_bits(got[:n], out0 + res if acc else res), ("burst", n, acc)
        for amp in (3.1e-14, -2.7e-14):
            out = _guarded(n, out0)
            _cabi.check(L.ptar_memory_delay(out.data_ptr(), t_d.data_ptr(), amp, t0, acc, n, s))
            with np.errstate(invalid="ignore"):
                res = np.where(t < t0, 0.0, amp * (t - t0))
            got = _np(out)
            assert _guards_ok(out, n)
            assert _same_bits(got[:n], out0 + res if acc else res), ("memory", n, acc, amp)
