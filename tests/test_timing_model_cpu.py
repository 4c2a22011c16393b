"""CPU tests of the timing-model fit (``PulsarBatch.set_timing_model``): the host statics of ``plan()`` against an
SVD least-squares oracle (tests/timing_oracle.py), their layout on the packed axis, and the argument checks."""
import numpy as np
import pytest

from oracle import refnumpy as O
from tests import timing_oracle as TO


def _psrs(seed=5, sizes=(37, 130, 1500, 2100), missing_flag=True):
    """Pulsars with 3-4 backends (flag ``f``) and a few TOAs that lack the flag."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, n in enumerate(sizes):
        mjd = rng.uniform(53000.0, 58800.0, n)         # table order is NOT time order
        err = rng.uniform(0.1, 3.0, n)
        be = ["A", "B", "C", "D"][: 3 + (j % 2)]
        flags = [{"f": be[int(q)]} for q in rng.integers(0, len(be), n)]
        if missing_flag:
            for q in rng.choice(n, size=max(2, n // 50), replace=False):
                flags[q] = {}
        p = pulsar_from_arrays(f"P{j}", {"RAJ": 1.0 + j, "DECJ": 10.0 * j - 20.0}, mjd.astype(np.longdouble), err, flags=flags)
        make_ideal(p)
        out.append(p)
    return out


def _batch(psrs):
    from pta_replicator_b200.engine import PulsarBatch
    return PulsarBatch(psrs, plan_only=True)


def _project(b, tm, rows):
    """r - W^{-1/2} Q (Q^T W^{1/2} r) from the plan's statics (rows [R, ld], engine order)."""
    out = np.array(rows, dtype=float, copy=True)
    for i in range(b.n_psr):
        k = int(tm["k"][i])
        if k == 0:
            continue
        n, s = b.ntoa[i], b.toa_off[i]
        Q = tm["Q"][tm["q_off"][i]:tm["q_off"][i] + k * n].reshape(k, n)
        sw = tm["sqrtw"][s:s + n]
        seg = out[:, s:s + n]
        out[:, s:s + n] = seg - ((seg * sw) @ Q.T) @ Q / sw
    return out


def _oracle_rows(b, rows, spec):
    """Per pulsar in table order: the SVD oracle on the design matrix of ``spec[i]`` = dict(poly, jumps, extra, sigma)."""
    out = np.array(rows, dtype=float, copy=True)
    for i, p in enumerate(b.psrs):
        if spec[i] is None:
            continue
        poly, jumps, extra, sigma = (spec[i].get(key) for key in ("poly", "jumps", "extra", "sigma"))
        t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
        fv = [f.get(jumps) for f in p.toas.table["flags"]] if jumps else None
        M = TO.timing_design_matrix(t, poly, fv, extra)
        sig = p.toas.get_errors().to("s").value if sigma is None else sigma
        s, n, o = b.toa_off[i], b.ntoa[i], b.order[i]
        tab = np.empty((rows.shape[0], n))
        tab[:, o] = rows[:, s:s + n]
        post = TO.postfit_lstsq(tab, M, sig)
        out[:, s:s + n] = post[:, o]
    return out


def _annual(p):
    t = np.asarray(p.toas.table["tdbld"], dtype=float) * 86400.0
    w = 2 * np.pi / (365.25 * 86400.0)
    return np.stack([np.sin(w * t), np.cos(w * t)], axis=1)


CASES = {
    "offset": lambda psrs: [dict(poly=0)] * len(psrs),
    "linear": lambda psrs: [dict(poly=1)] * len(psrs),
    "spin": lambda psrs: [dict(poly=2)] * len(psrs),
    "spin_jumps": lambda psrs: [dict(poly=2, jumps="f")] * len(psrs),
    "jumps_only": lambda psrs: [dict(poly=None, jumps="f")] * len(psrs),
    "linear_annual_unweighted": lambda psrs: [dict(poly=1, extra=_annual(p), sigma=np.ones(p.toas.ntoas)) for p in psrs],
    "mixed_with_modelless": lambda psrs: [dict(poly=2, jumps="f"), None, dict(poly=0, extra=_annual(psrs[2])), None],
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_projection_from_plan_statics_matches_svd_oracle(case):
    psrs = _psrs()
    spec = CASES[case](psrs)
    b = _batch(psrs)
    for i, sp in enumerate(spec):
        if sp is not None:
            b.set_timing_model(i, **sp)
    tm = b.plan()["tm"]
    rng = np.random.default_rng(11)
    rows = np.zeros((5, b.ld))
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        rows[:, s:s + n] = 1e-6 * rng.standard_normal((5, n)) + 3e-6 * rng.standard_normal((5, 1))
    got = _project(b, tm, rows)
    ref = _oracle_rows(b, rows, spec)
    for i in range(b.n_psr):
        s, n = b.toa_off[i], b.ntoa[i]
        if spec[i] is None:
            assert np.array_equal(got[:, s:s + n], rows[:, s:s + n])
            continue
        rms = np.sqrt(np.mean(ref[:, s:s + n] ** 2))
        err = np.max(np.abs(got[:, s:s + n] - ref[:, s:s + n])) / rms
        assert err < 1e-13, (case, i, err)
        # the fit removed something: post-fit differs from pre-fit
        assert np.max(np.abs(got[:, s:s + n] - rows[:, s:s + n])) > 1e-3 * rms


def test_q_is_orthonormal_and_padding_is_zero():
    psrs = _psrs()
    b = _batch(psrs)
    b.set_timing_model(0, poly=2, jumps="f")
    b.set_timing_model(2, poly=1, extra=_annual(psrs[2]), sigma=np.linspace(1e-7, 2e-6, psrs[2].toas.ntoas))
    tm = b.plan()["tm"]
    assert list(tm["k"]) == [2 + 1 + 3, 0, 2 + 2, 0]          # 3 backends + "no flag" group, one dropped
    assert tm["kmax"] == 6
    assert tm["Q"].size == 6 * b.ntoa[0] + 4 * b.ntoa[2]
    for i in (0, 2):
        k, n = int(tm["k"][i]), b.ntoa[i]
        Q = tm["Q"][tm["q_off"][i]:tm["q_off"][i] + k * n].reshape(k, n)
        assert np.max(np.abs(Q @ Q.T - np.eye(k))) < 1e-13
    live = np.zeros(b.ld, dtype=bool)
    for i in (0, 2):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    assert np.all(tm["sqrtw"][~live] == 0) and np.all(tm["sqrtw"][live] > 0)
    tiles = tm["tiles"]
    assert set(tiles[:, 5]) == {0, 2}
    for i in (0, 2):
        mine = tiles[tm["tile0"][i]:tm["tile0"][i] + tm["n_tile"][i]]
        assert np.all(mine[:, 5] == i) and mine[:, 1].sum() == b.ntoa[i] and np.all(mine[:, 1] <= 1024)
        assert np.all(mine[:, 0] % 4 == 0) and np.all(mine[:, 0] - mine[:, 2] == b.toa_off[i])
    assert tm["n_tile"][1] == 0 and tm["n_tile"][3] == 0


def test_offset_fit_is_the_weighted_mean():
    psrs = _psrs(sizes=(50, 70))
    b = _batch(psrs)
    for i in range(2):
        b.set_timing_model(i, poly=0)
    tm = b.plan()["tm"]
    rng = np.random.default_rng(3)
    row = np.zeros((1, b.ld))
    for i in range(2):
        row[0, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = 2e-7 + 1e-7 * rng.standard_normal(b.ntoa[i])
    got = _project(b, tm, row)
    for i in range(2):
        s, n = b.toa_off[i], b.ntoa[i]
        ref = O.weighted_mean_residual(row[0, s:s + n], b.err_s[i])
        assert np.max(np.abs(got[0, s:s + n] - ref)) < 1e-13 * np.sqrt(np.mean(ref**2))


def test_empty_model_clears_and_setter_drops_compiled_state():
    b = _batch(_psrs())
    b.set_timing_model(1, poly=2)
    assert b.plan()["tm"] is not None
    b._compiled = object()
    b.set_timing_model(1, poly=None)
    assert b._compiled is None
    assert b.plan()["tm"] is None


def test_value_errors():
    psrs = _psrs()
    b = _batch(psrs)
    n0 = psrs[0].toas.ntoas
    with pytest.raises(ValueError, match="rank-deficient"):
        b.set_timing_model(0, poly=2, extra=np.ones(n0))             # duplicates the offset
    with pytest.raises(ValueError, match="rank-deficient"):
        b.set_timing_model(0, poly=None, extra=np.zeros((n0, 1)))
    with pytest.raises(ValueError, match="at most 32"):
        b.set_timing_model(3, poly=2, extra=np.random.default_rng(0).standard_normal((psrs[3].toas.ntoas, 30)))
    small = _batch(_psrs(sizes=(20, 40)))
    with pytest.raises(ValueError, match="fewer columns than TOAs"):
        small.set_timing_model(0, poly=2, extra=np.random.default_rng(0).standard_normal((20, 17)))
    for bad in (np.ones(n0 - 1), -np.ones(n0), np.zeros(n0), np.r_[np.ones(n0 - 1), np.nan], np.r_[np.ones(n0 - 1), np.inf]):
        with pytest.raises(ValueError, match="sigma"):
            b.set_timing_model(0, poly=2, sigma=bad)
    for bad in (np.ones((n0 + 1, 2)), np.ones((2, n0)), np.ones((n0, 2, 1)), np.full((n0, 1), np.nan)):
        with pytest.raises(ValueError, match="extra"):
            b.set_timing_model(0, poly=2, extra=bad)
    with pytest.raises(ValueError, match="poly"):
        b.set_timing_model(0, poly=-1)
    assert b._tm is None or all(m is None for m in b._tm)               # nothing half-registered
