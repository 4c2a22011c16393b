"""CPU tests of the Fp-statistic's host statics (``PulsarBatch.set_fp_statistic``, ``plan()["fp"]``) against the dense
oracle (tests/fp_oracle.py), the whitening identities, the default grid, independence from the optimal statistic's
statics and every argument check.  ``plan_only`` batches: the 3 ``partim_small`` pulsars and the 4-pulsar synthetic case
of tests/test_optimal_statistic_cpu.py."""
import numpy as np
import pytest

from tests import fp_oracle as FO
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# Woodbury (host statics) and the dense null-space solve (oracle) round differently; the optimal statistic's bound.
TOL = 1e-10
NF = 12


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / np.max(np.abs(b)))


def _ct(b, pf, i):
    from pta_replicator_b200.engine import fp_whitened_basis
    return fp_whitened_basis(pf, b.toa_off[i], b.ntoa[i])


def _live(b):
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    return live


CASES = [(src, tm, common) for src in ("small", "synthetic") for tm in (False, True) for common in (None, -14.5)]


@pytest.mark.parametrize("src,tm,common", CASES)
def test_statics_match_dense_oracle(src, tm, common):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    b.set_fp_statistic(n_freqs=NF, log10_A_common=common)
    pf = b.plan()["fp"]
    S = FO.statics(b, pf["freqs"], log10_A_common=common, models=_models(b) if tm else None)
    worst = dict(Ct=max(_rel(_ct(b, pf, i), S["Ct"][i]) for i in range(b.n_psr)),
                 M=max(_rel(pf["M"][i], S["M"][i]) for i in range(b.n_psr)))
    rows = np.random.default_rng(1).standard_normal((5, b.ld)) * 1e-6
    rows[:, ~_live(b)] = 0
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ _ct(b, pf, i) for i in range(b.n_psr)], axis=1)
    fp = 0.5 * np.sum(X.reshape(5, b.n_psr, NF, 2) ** 2, axis=(1, 3))
    worst["Fp"] = _rel(fp, FO.fp_of_rows(b, S, rows))
    # whitening: C~_a(f)^T P_a C~_a(f) = I_2
    wh = 0.0
    for i in range(b.n_psr):
        Ct = _ct(b, pf, i)
        G = Ct.T @ S["P"][i] @ Ct
        for f in range(NF):
            wh = max(wh, float(np.max(np.abs(G[2 * f:2 * f + 2, 2 * f:2 * f + 2] - np.eye(2)))))
    worst["whitening"] = wh
    print(f"\n[fp statics] {src} tm={tm} common={common}: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert max(worst.values()) < TOL, worst
    # layout: alignment slots and padding columns carry no weight
    assert np.all(pf["Ct"][:, ~_live(b), :] == 0)
    full = np.concatenate([_ct(b, pf, i) for i in range(b.n_psr)])
    assert full.shape[1] == 2 * NF and pf["n_cb"] == 1


@pytest.mark.parametrize("src", ["small", "synthetic"])
def test_whitened_basis_annihilates_the_timing_model(src):
    b = _batch(_small() if src == "small" else _synthetic(), tm=True)
    b.set_fp_statistic(n_freqs=40)
    pf = b.plan()["fp"]
    M = _models(b)
    worst = 0.0
    for i in range(b.n_psr):
        Ct = _ct(b, pf, i)
        worst = max(worst, float(np.max(np.abs(Ct.T @ M[i])) / (np.linalg.norm(Ct) * np.linalg.norm(M[i]))))
    print(f"\n[fp statics] {src}: max |C~^T M| / (|C~| |M|) = {worst:.1e}")
    assert worst < 1e-17


def test_layout_spans_column_blocks_and_rotates_odd_toas():
    b = _batch(_synthetic(), tm=True)
    b.set_fp_statistic(n_freqs=40)          # 80 columns: 2 blocks of 64, the second one padded
    pf = b.plan()["fp"]
    assert pf["Ct"].shape == (2, b.ld, 64) and pf["n_cb"] == 2
    S = FO.statics(b, pf["freqs"], models=_models(b))
    i = 1
    s, n = b.toa_off[i], b.ntoa[i]
    raw = pf["Ct"][:, s:s + n, :]
    for k in (0, 1, 2, 3):                   # both parities of the packed index
        want = np.zeros(128)
        want[:80] = S["Ct"][i][k]
        got = raw[:, k, :].copy()
        if (s + k) & 1:
            got = np.roll(got, -8, axis=-1)
        assert np.allclose(got.ravel(), want, rtol=0, atol=1e-10 * np.max(np.abs(want)))
    assert np.all(pf["Ct"][1, :, :][:, np.r_[16:64]][::2] == 0)       # padding columns 80..127 of even TOAs
    assert np.array_equal(pf["psr_order"], np.argsort(-np.asarray(b.ntoa), kind="stable"))


def test_default_grid_and_outputs():
    b = _batch(_synthetic())
    Tspan = max(t.max() for t in b.t_tdb) - min(t.min() for t in b.t_tdb)
    b.set_fp_statistic(n_freqs=7)
    pf = b.plan()["fp"]
    assert np.array_equal(pf["freqs"], np.arange(1, 8) / Tspan) and pf["n_freq"] == 7
    assert pf["M"].shape == (4, 7, 2, 2) and np.array_equal(pf["M"], pf["M"].transpose(0, 1, 3, 2))
    assert b.fp_setup_s is not None and b.fp_setup_s >= 0 and pf["setup_s"] == b.fp_setup_s
    b.set_fp_statistic(n_freqs=5, Tspan=3e8)
    assert np.array_equal(b.plan()["fp"]["freqs"], np.arange(1, 6) / 3e8)
    f = np.array([3e-9, 1e-8, 2.5e-8])
    b.set_fp_statistic(freqs=f)
    assert np.array_equal(b.plan()["fp"]["freqs"], f)


def test_registration_is_independent_of_the_optimal_statistic():
    b = _batch(_synthetic(), tm=True)
    assert b.plan()["fp"] is None
    b.set_optimal_statistic(orfs=("hd",))
    b.set_os_null("phase_shift", n=8)
    plain = b.plan()
    b.set_fp_statistic(n_freqs=10, log10_A_common=-14.5)
    both = b.plan()
    for key in ("os", "os_null"):
        for k, v in plain[key].items():
            if isinstance(v, np.ndarray):
                assert np.array_equal(v, both[key][k]), (key, k)
    assert b._os_null is not None and both["fp"] is not None
    b.set_optimal_statistic(orfs=("hd",))     # re-registering the OS leaves the Fp registration alone
    assert b.plan()["fp"] is not None


def test_device_calls_of_a_plan_only_batch_raise():
    from pta_replicator_b200._cabi import PtarError
    b = _batch(_synthetic())
    b.set_fp_statistic(n_freqs=4)
    with pytest.raises(PtarError):
        b.fp_statistic(8)
    with pytest.raises(PtarError):
        b.fp_statistic_of(np.zeros((4, b.ld)))


def test_value_errors():
    psrs = _synthetic()
    b = _batch(psrs)
    for bad, msg in (([], "empty"), ([1e-8, np.nan], "finite and positive"), ([1e-8, -1e-9], "finite and positive"),
                     ([0.0], "finite and positive"), ([1e-8, 2e-8, 1e-8], "duplicates"),
                     (np.arange(1, 258) * 1e-9, "at most 256")):
        with pytest.raises(ValueError, match=msg):
            b.set_fp_statistic(freqs=bad)
    for bad in (0, 257, 2.5, True):
        with pytest.raises(ValueError, match="n_freqs"):
            b.set_fp_statistic(n_freqs=bad)
    for bad in (0.0, -1.0, np.nan, np.inf):
        with pytest.raises(ValueError, match="Tspan"):
            b.set_fp_statistic(Tspan=bad)
    with pytest.raises(ValueError, match="log10_A_common"):
        b.set_fp_statistic(log10_A_common=np.nan)
    with pytest.raises(ValueError, match="gamma_common"):
        b.set_fp_statistic(gamma_common=np.inf)
    with pytest.raises(ValueError, match="components_common"):
        b.set_fp_statistic(components_common=0)
    assert b._fp is None                      # nothing was registered by a failed call
    # a pulsar without white noise
    nw = _batch(psrs, white=False)
    nw.set_white(0, efac=1.0)
    nw.set_fp_statistic(n_freqs=4)
    with pytest.raises(ValueError, match="set_white"):
        nw.plan()
    # zero white variance on some TOAs
    zw = _batch(psrs)
    zw.set_white(2, efac=np.array([1.0, 0.0, 1.0]), log10_equad=np.array([-np.inf, -np.inf, -np.inf]), flagid="f",
                 flags=["A", "B", "C"])
    zw.set_fp_statistic(n_freqs=4)
    with pytest.raises(ValueError, match="zero white-noise variance"):
        zw.plan()
    # a timing model that contains the sinusoid at grid frequency 3 of pulsar 1 absorbs it
    ab = _batch(psrs)
    Tspan = max(t.max() for t in ab.t_tdb) - min(t.min() for t in ab.t_tdb)
    t = np.asarray(psrs[1].toas.table["tdbld"], dtype=float) * 86400.0
    arg = 2 * np.pi * 3 / Tspan * t
    ab.set_timing_model(1, poly=2, extra=np.stack([np.sin(arg), np.cos(arg)], axis=1))
    ab.set_fp_statistic(n_freqs=6)
    with pytest.raises(ValueError, match=r"pulsar 1 \(S1\) at f = .* \(frequency index 2\) is not safely positive definite"):
        ab.plan()
