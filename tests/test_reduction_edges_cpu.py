"""CPU tests of the extended-precision reference of the per-realization reductions (tests/reduction_reference.py): the
reference is exact enough, its bounds reject subtly wrong results, the edge batches reach every kernel variant the GPU
sweep claims, and Q(P, x) restated in numpy matches an independent evaluation."""
from fractions import Fraction

import numpy as np
import pytest

from tests import reduction_reference as RR

U = RR.U


def _fsum_prod(a, b):
    return sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a, b)), Fraction(0))


def _err(h, l, exact):
    return abs(Fraction(float(h)) + Fraction(float(l)) - exact)


@pytest.mark.parametrize("dot2", [False, True] if RR.LONG else [True])
def test_reference_is_exact_to_well_below_its_bound(dot2):
    """xmatmul / xsum_prod / xscale / xdiv against Fraction sums: error <= 1e-3 of the bound they serve."""
    rng = np.random.default_rng(1)
    worst = 0.0
    for n in (1, 5, 64, 193):
        A = rng.standard_normal((3, n)) * np.exp(rng.uniform(-20, 20, (3, n)))
        B = rng.standard_normal((n, 2))
        h, l = RR.xmatmul(A, B, dot2=dot2)
        bound = RR.gamma(n + 8) * (np.abs(A) @ np.abs(B))
        for r in range(3):
            for j in range(2):
                ex = _fsum_prod(A[r], B[:, j])
                worst = max(worst, float(_err(h[r, j], l[r, j], ex)) / bound[r, j])
        h2, l2 = RR.xsum_prod(A, 0.0, A[:, ::-1], 0.0, dot2=dot2)
        b2 = RR.gamma(n + 8) * np.sum(np.abs(A * A[:, ::-1]), axis=-1)
        for r in range(3):
            worst = max(worst, float(_err(h2[r], l2[r], _fsum_prod(A[r], A[r, ::-1]))) / b2[r])
        s, t = rng.standard_normal(2)
        sh, sl = RR.xscale(h[0, 0], l[0, 0], s)
        ex = (Fraction(float(h[0, 0])) + Fraction(float(l[0, 0]))) * Fraction(float(s))
        worst = max(worst, float(_err(sh, sl, ex)) / (U * abs(float(ex))))
        dh, dl = RR.xdiv(h[0, 0], l[0, 0], t)
        ex = (Fraction(float(h[0, 0])) + Fraction(float(l[0, 0]))) / Fraction(float(t))
        worst = max(worst, float(_err(dh, dl, ex)) / (U * abs(float(ex))))
    print(f"\n[reference] dot2={dot2}: worst error / bound {worst:.1e}")
    assert worst <= 1e-3


def _fp64_projection(rows, B, s, n):
    return rows[:, s:s + n] @ B[s:s + n]


def _case(seed=2, R=70, n=130, c=8):
    rng = np.random.default_rng(seed)
    ld = 4 * ((n + 3) // 4) + 4
    rows = np.zeros((R, ld))
    rows[:, :n] = rng.standard_normal((R, n))
    B = np.zeros((ld, c))
    B[:n] = rng.standard_normal((n, c))
    return rows, B, n


def test_fp64_projection_passes_and_mutations_fail():
    """numpy's own fp64 product is within the bound; each subtly wrong variant is not."""
    rows, B, n = _case()
    h, l, bound, terms = RR.projection(rows, B, 0, n)
    ref = dict(hi=h, lo=l, bound=bound, terms=terms)
    good = _fp64_projection(rows, B, 0, n)
    assert RR.check(good, ref, "fp64")[0] <= 1.0
    mutants = {}
    # one TOA dropped from the sum
    mutants["dropped TOA"] = good - np.outer(rows[:, n - 1], B[n - 1])
    # an alignment slot that holds data and is summed (with the coefficients of the pulsar's last TOA)
    poison = rows.copy()
    poison[:, n] = rows[:, n - 1]
    mutants["alignment slot summed"] = good + np.outer(poison[:, n], B[n - 1])
    # the output of row r written to row r + 1 of a ragged block (rows 64.. of 70)
    m = good.copy()
    m[65] = good[64]
    mutants["row r -> r + 1"] = m
    # column block cb read with the offset of cb - 1 (blocks of 4 columns)
    m = good.copy()
    m[:, 4:8] = good[:, 0:4]
    mutants["column block offset"] = m
    # a k-quarter lost: TOAs 16..31 of every 64-TOA chunk
    lost = np.array([i for i in range(n) if 16 <= i % 64 < 32])
    mutants["k-quarter lost"] = good - rows[:, lost] @ B[lost]
    for name, mu in mutants.items():
        with pytest.raises(AssertionError):
            RR.check(mu, ref, name)


def test_fp_reduce_pulsar_counted_twice_fails():
    rng = np.random.default_rng(3)
    P, n, Nf = 5, 40, 3
    seg_off, seg_len = [48 * a for a in range(P)], [n] * P
    rows = np.zeros((4, 48 * P))
    Ct = []
    for a in range(P):
        rows[:, seg_off[a]:seg_off[a] + n] = rng.standard_normal((4, n))
        Ct.append(rng.standard_normal((n, 2 * Nf)))
    ref = RR.fp_statistic(Ct, seg_off, seg_len, rows)
    amps = np.stack([rows[:, s:s + n] @ C for s, C in zip(seg_off, Ct)], axis=1)
    Fp = 0.5 * np.sum(amps.reshape(4, P, Nf, 2) ** 2, axis=(1, 3))
    RR.check(amps, ref["amps"], "amps")
    RR.check(Fp, ref["Fp"], "Fp")
    with pytest.raises(AssertionError):
        RR.check(Fp + 0.5 * np.sum(amps[:, 2].reshape(4, Nf, 2) ** 2, axis=-1), ref["Fp"], "pulsar 2 twice")


def test_timing_reference_bound_holds_where_the_fit_cancels():
    """Rows that lie almost in the model's column space (post-fit 1e-6 of pre-fit): numpy's fp64 fit passes the bound,
    a fit that forgets the 1/sqrt(w) factor or drops a column does not."""
    rng = np.random.default_rng(4)
    n, k = 37, 3
    t = np.sort(rng.uniform(0, 1, n))
    M = np.stack([t**d for d in range(k)], axis=1)
    sw = 1.0 / rng.uniform(0.5, 2.0, n)
    Q, _ = np.linalg.qr(M * sw[:, None])
    rows = np.zeros((5, 40))
    rows[:, :n] = (rng.standard_normal((5, k)) @ M.T) + 1e-6 * rng.standard_normal((5, n))
    T = dict(k=np.array([k]), q_off=np.array([0]), Q=Q.T.ravel(), sqrtw=np.r_[sw, np.zeros(3)], seg_off=np.array([0]),
             seg_len=np.array([n]))
    ref = RR.timing_fit(T, rows)
    r = rows[:, :n]
    c = (r * sw) @ Q
    good = rows.copy()
    good[:, :n] = r - (c @ Q.T) * (1.0 / sw)
    RR.check(good, ref, "fp64 fit")
    bad = rows.copy()
    bad[:, :n] = r - (c[:, :2] @ Q[:, :2].T) / sw
    with pytest.raises(AssertionError):
        RR.check(bad, ref, "column dropped")
    bad = good.copy()
    bad[:, n] = 1.0                                  # a padding slot written
    with pytest.raises(AssertionError):
        RR.check(bad, ref, "padding written")


# ------------------------------------------------------------------ coverage by construction
def test_edge_batches_reach_every_variant():
    from pta_replicator_b200 import _cabi
    b = RR.edge_batch(RR.EDGE_NTOAS, seed=0, plan_only=True)
    n = np.asarray(b.ntoa)
    assert {1, 2, 3} <= set((n % 4).tolist())                         # pulsars with n mod 4 in {1, 2, 3}
    assert np.any(n < 64) and np.all(n[n < 8] % 4 != 0)               # the only chunk partial
    assert np.any((n > 3 * 64) & (n % 64 != 0))                       # >= 4 chunks, partial last: the ring wraps
    assert np.any(-(-n // _cabi.TILE_TOAS) >= 3)                      # a pulsar split into >= 3 tiles
    ncp = set()
    for K, kind, R in RR.os_cases():
        b.set_optimal_statistic(components=K, orfs=RR.templates(b.n_psr, kind))
        po = b._plan_os()
        ncp.add(po["ncp"])
        assert po["orf"].shape[0] == (1 if kind == "hd" else 4)
    assert ncp == {8, 16, 24, 32}
    assert {R for _, _, R in RR.os_cases()} >= {1, 3, 63, 64, 65, 130}
    ncb, last = set(), set()
    for nf, R in RR.fp_cases():
        nf = 20 if nf == "unsorted" else nf
        ncb.add(-(-2 * nf // 64))
        last.add((2 * nf) % 64 == 0)
    assert ncb == {1, 2, 4, 8} and last == {True, False}
    buckets = {4 if k <= 4 else 8 if k <= 8 else 16 if k <= 16 else 32 for k in RR.TM_KMAX}
    assert buckets == {4, 8, 16, 32}
    cols, kdp = set(), []
    for method, nn, K, P, R in RR.null_cases():
        nc = nn + 1
        cols.add("<64" if nc < 64 else "=64" if nc == 64 else ">64")
        kd = P * (P - 1) // 2 * (2 * K if method == "phase_shift" else 1)
        kdp.append(-(-kd // 32) * 32 > kd)
    assert cols == {"<64", "=64", ">64"} and any(kdp)
    assert {P for *_, P, _ in RR.null_cases()} == {2, 3, 24}


def test_edge_batch_statics_plan():
    """The plan of an edge batch holds (no absorbed frequency; every timing model full rank) for the Fp grids."""
    b = RR.edge_batch((5, 6, 7, 64, 65, 193), seed=5, plan_only=True)
    b.set_fp_statistic(n_freqs=33)
    pf = b._plan_fp()
    assert pf["n_cb"] == 2 and pf["Ct"].shape[1] == b.ld
    for k in RR.TM_KMAX:
        poly, ex = RR.tm_columns(b, 5, k)
        b.set_timing_model(5, poly=poly, extra=ex)
        assert b._tm[5]["k"] == k


# ------------------------------------------------------------------ Q(P, x)
@pytest.mark.parametrize("P", [1, 2, 3, 24, 67, 256])
def test_q_int_matches_independent_evaluation(P):
    xs = np.unique(np.r_[0.0, 1e-300, 1e-8, 0.5, 1.0, P - 1, P, P + 0.5, np.linspace(0, 4 * P + 400, 257), 745.5, 800.0,
                         P + np.sqrt(P) * np.linspace(-4, 4, 33)])
    xs = xs[xs >= 0]
    try:
        import mpmath
        mpmath.mp.dps = 40
        ref = np.array([float(mpmath.gammainc(P, float(x), mpmath.inf, regularized=True)) for x in xs])
        src = "mpmath"
    except ImportError:
        from scipy.special import gammaincc
        ref = gammaincc(P, xs)
        src = "scipy"
    got = RR.q_int(P, xs)
    keep = ref >= 1e-300
    rel = np.abs(got[keep] - ref[keep]) / ref[keep]
    print(f"\n[Q] P={P}: worst relative error {rel.max():.1e} against {src} over {keep.sum()} points, x up to {xs.max():.0f}")
    assert rel.max() <= 1e-12
    assert got[0] == 1.0 and np.all(got[~keep] <= 1e-290)
    ld = RR.q_int(P, xs, np.longdouble).astype(float)
    assert np.max(np.abs(ld[keep] - ref[keep]) / ref[keep]) <= 1e-12
