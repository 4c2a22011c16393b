"""CPU tests of the sine-Gaussian burst search's host statics (``PulsarBatch.set_burst_statistic``, ``plan()["burst"]``)
against the dense oracle (tests/burst_oracle.py): the factored device arithmetic (N^-1 r per ECORR run, z, W^T N^-1 r -
H^T z) against dense P_a^{-1} W, the windows and the unseen rule, the coherent bound, the default bank, every argument
and plan-time check, the independence of the other statistics' statics and the batch ``add_noise_transient``.
``plan_only`` batches: the 3 ``partim_small`` pulsars and the 4-pulsar synthetic case of tests/test_optimal_statistic_cpu.py."""
import numpy as np
import pytest

from tests import burst_oracle as UO
from tests import fe_oracle as EO
from tests.test_fe_statistic_cpu import _live_rows
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# Factored (host statics + device arithmetic emulated in numpy) against dense null-space solves: both fp64.  Measured on
# these cases: M <= 1.2e-14, W^T P^-1 r <= 3.7e-14 relative to the largest entry; the bound leaves room for other BLAS
# builds.
TOL = 1e-10
# Pre-fit rows whose timing-model component is 1e2 x the noise: W^T N^-1 r and H^T z are each ~1e2 x the answer and
# cancel (the dense G-projection never forms them), so the factored form keeps ~2 digits fewer.  Measured <= 7.4e-13.
TOL_PREFIT = 1e-10
CASES = [(src, tm, common) for src in ("small", "synthetic") for tm in (False, True) for common in (None, -14.5)]


def _bank(b, n=12, seed=0):
    """An explicit bank across the batch's span: Q in {3, 6}, f0 from 1 / Tspan to 30 / Tspan."""
    rng = np.random.default_rng(seed)
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    Tspan = (last - first) * 86400
    return rng.uniform(first, last, n), rng.uniform(1.0, 30.0, n) / Tspan, rng.choice([3.0, 6.0], n)


def _prefit_rows(b, models, R=4, seed=2):
    """Noise-level rows plus a timing-model component 1e2 x larger on every pulsar."""
    rows = _live_rows(b, R, seed=seed)
    rng = np.random.default_rng(seed + 1)
    for i, Mt in enumerate(models):
        s, n = b.toa_off[i], b.ntoa[i]
        c = Mt @ rng.standard_normal((Mt.shape[1], R))
        rows[:, s:s + n] += 1e2 * 1e-6 * (c / np.sqrt(np.mean(c * c, axis=0))).T
    return rows


@pytest.mark.parametrize("src,tm,common", CASES)
def test_factored_statics_match_dense_oracle(src, tm, common):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    t0, f0, Q = _bank(b)
    b.set_burst_statistic(t0_mjd=t0, f0=f0, Q=Q, nside=1, log10_A_common=common)
    pb = b.plan()["burst"]
    models = _models(b) if tm else None
    S = UO.statics(b, pb["templates"], log10_A_common=common, models=models)
    assert np.array_equal(pb["seen"], S["seen"])
    for i in range(b.n_psr):
        assert np.array_equal(pb["win"][i], UO.windows(b, i, pb["templates"]))
    seen = S["seen"][..., None, None]
    dm = float(np.max(np.abs(np.where(seen, pb["M"] - S["M"], 0))) / np.max(np.abs(S["M"])))
    rows = _live_rows(b, 5)
    N, X = UO.emulate(b, pb, rows)
    ref = UO.dense_n(b, S, rows)
    dn = float(np.max(np.abs(np.where(seen[None, ..., 0], N - ref, 0))) / np.max(np.abs(ref)))
    print(f"\n[burst statics] {src} tm={tm} common={common}: seen {int(pb['seen'].sum())}/{pb['seen'].size}, M {dm:.1e}, "
          f"W^T P^-1 r {dn:.1e}")
    assert dm < TOL and dn < TOL
    assert np.all(X[:, ~pb["seen"]] == 0)
    if tm:
        rows = _prefit_rows(b, models)
        N, _ = UO.emulate(b, pb, rows)
        ref = UO.dense_n(b, S, rows)
        dp = float(np.max(np.abs(np.where(seen[None, ..., 0], N - ref, 0))) / np.max(np.abs(ref)))
        print(f"[burst statics] pre-fit rows (timing model 1e2 x noise): {dp:.1e}")
        assert dp < TOL_PREFIT


def test_coherent_bound_and_windows():
    b = _batch(_synthetic(), tm=True)
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    Tspan = (last - first) * 86400
    # a template whose window holds the whole span, beside two of the bank
    t0 = np.array([0.5 * (first + last), first + 0.3 * (last - first), first + 0.7 * (last - first)])
    f0 = np.array([2.0 / Tspan, 12.0 / Tspan, 20.0 / Tspan])
    Q = np.array([8.0, 4.0, 4.0])
    b.set_burst_statistic(t0_mjd=t0, f0=f0, Q=Q, nside=1)
    pb = b.plan()["burst"]
    whole = int(np.argmax(pb["tau"]))
    assert all(tuple(pb["win"][i, whole]) == (0, b.ntoa[i]) for i in range(b.n_psr))
    for i in range(b.n_psr):
        assert np.array_equal(pb["win"][i], UO.windows(b, i, pb["templates"]))
    # block ranges: the union of the block's windows, lo aligned down to 4
    for i in range(b.n_psr):
        ne = pb["win"][i, :, 1] > pb["win"][i, :, 0]
        assert pb["blk"][i, 0, 0] == pb["win"][i, ne, 0].min() // 4 * 4 and pb["blk"][i, 0, 1] == pb["win"][i, ne, 1].max()
    # B <= 1/2 sum_a |X^_a|^2 at every cell (explicit 4 x 4 solves of the oracle)
    rows = _live_rows(b, 6, seed=5)
    _, X = UO.emulate(b, pb, rows)
    ok = pb["seen"].sum(axis=0) >= 2
    B, _ = UO.coherent(pb, X[:, :, ok], EO.antenna(b, pb["sky"]))
    assert np.all(B <= 0.5 * np.sum(X[:, :, ok] ** 2, axis=(1, 3))[:, :, None] * (1 + 1e-12))


@pytest.mark.parametrize("src", ["small", "synthetic"])
def test_default_bank(src):
    b = _batch(_small() if src == "small" else _synthetic(), tm=True)
    b.set_burst_statistic(nside=1)
    reg = b._burst["templates"]
    tau = reg[:, 2] / (2 * np.pi * reg[:, 1])
    assert np.all(np.diff(tau) >= 0)                                  # held sorted by (tau, t0, Q)
    Tspan = b._array_tspan(None)
    assert np.allclose(np.unique(np.round(reg[:, 1] * Tspan, 6)), np.arange(2, 21))
    assert set(np.unique(reg[:, 2])) == {4.0, 8.0}
    first, last = min(m.min() for m in b.mjd), max(m.max() for m in b.mjd)
    assert reg[:, 0].min() >= first and reg[:, 0].max() <= last
    pb = b.plan()["burst"]
    assert np.all(pb["seen"].sum(axis=0) >= 2) and pb["n_tmpl"] <= len(reg)
    assert pb["linv"].shape == (pb["n_tmpl"], 32, 10) and pb["Lf"].shape == (pb["n_tmpl"], b.n_psr, 3)
    assert b.burst_setup_s == pb["setup_s"]


def test_value_errors():
    psrs = _synthetic()
    from pta_replicator_b200.engine import PulsarBatch
    with pytest.raises(ValueError, match="at least 2 pulsars"):
        PulsarBatch(psrs[:1], plan_only=True).set_burst_statistic()
    b = _batch(psrs)
    t0, f0, Q = _bank(b, 4)
    for kw, msg in [(dict(t0_mjd=[], f0=[], Q=[]), "empty"),
                    (dict(t0_mjd=t0, f0=f0[:3], Q=Q), "equal lengths"),
                    (dict(t0_mjd=t0, f0=None), "needs t0_mjd, f0 and Q"),
                    (dict(t0_mjd=[np.nan] + list(t0[1:]), f0=f0, Q=Q), "finite"),
                    (dict(t0_mjd=t0, f0=-f0, Q=Q), "positive"),
                    (dict(t0_mjd=t0, f0=f0, Q=np.zeros(4)), "positive"),
                    (dict(t0_mjd=np.r_[t0, t0[:1]], f0=np.r_[f0, f0[:1]], Q=np.r_[Q, Q[:1]]), "duplicates"),
                    (dict(t0_mjd=np.arange(4097.0) + 53000, f0=np.full(4097, 1e-8), Q=4.0), "at most 4096"),
                    (dict(Q=(4.0, -1.0)), "Q must be"),
                    (dict(n_f0=0), "n_f0"),
                    (dict(nside=3), "nside"),
                    (dict(sky=np.zeros((3, 3))), "sky"),
                    (dict(log10_A_common=np.inf), "log10_A_common"),
                    (dict(gamma_common=np.nan), "gamma_common")]:
        with pytest.raises(ValueError, match=msg):
            b.set_burst_statistic(**kw)
    big = PulsarBatch(psrs * 33, plan_only=True)
    with pytest.raises(ValueError, match="at most 128 pulsars"):
        big.set_burst_statistic()
    # plan time: white noise missing; an explicit template that only one pulsar sees (M4 singular), naming it
    nw = _batch(psrs, white=False)
    nw.set_burst_statistic(t0_mjd=t0, f0=f0, Q=Q)
    with pytest.raises(ValueError, match="white noise"):
        nw.plan()
    lone = float(b.mjd[0][3])
    others = np.concatenate([m for m in b.mjd[1:]])
    assert np.min(np.abs(others - lone)) * 86400 > 60
    b.set_burst_statistic(t0_mjd=[lone], f0=[1.0 / 5.0], Q=[4.0], nside=1)
    with pytest.raises(ValueError, match=r"M4\(j, s\) at template 0 .* sky point 0"):
        b.plan()


def test_other_plans_unchanged():
    b = _batch(_synthetic(), tm=True)
    b.set_fp_statistic(n_freqs=6, log10_A_common=-14.5)
    b.set_fe_statistic(nside=1)
    b.set_bwm_statistic(n_epochs=5, nside=1)
    b.set_curn_likelihood(log10_A=np.linspace(-16, -13, 5), gamma=[3.0, 4.0], components=4)
    ref = b.plan()
    b.set_burst_statistic(nside=1)
    got = b.plan()
    assert got["burst"] is not None and ref["burst"] is None
    for key in ("fp", "fe", "bwm", "curn"):
        for k, v in ref[key].items():
            if k != "setup_s" and isinstance(v, np.ndarray):
                assert np.array_equal(v, got[key][k]), (key, k)


def test_batch_noise_transient_matches_drop_in(monkeypatch):
    from pta_replicator_b200 import deterministic
    psrs = _synthetic()
    b = _batch(psrs)
    t0 = float(np.median(b.mjd[2])) * 86400

    def wf(t):
        return 3e-7 * np.exp(-((t - t0) / 4e6) ** 2) * np.cos(2 * np.pi * 2e-7 * (t - t0))

    b.add_noise_transient(2, wf)
    seen = {}
    monkeypatch.setattr(deterministic, "_inject", lambda psr, name, params, seconds: seen.update({psr.name: seconds}))
    deterministic.add_noise_transient(psrs[2], wf)
    assert np.array_equal(b._det[2], seen[psrs[2].name][b.order[2]])
    assert all(not np.any(b._det[i]) for i in (0, 1, 3))


def test_default_bank_drops_templates_whose_m4_is_singular():
    """Two pulsars at one sky position observe the first half of the span, a third pulsar elsewhere the second half:
    an early template is seen by two pulsars whose antenna patterns are equal, so its M4 has rank 2 at every sky point.
    The default bank leaves such templates out and plans; an explicit bank with one of them is a plan-time error."""
    from pta_replicator_b200.engine import PulsarBatch
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(4)
    psrs = []
    for j, (ra, dec, lo, hi) in enumerate([(1.37, 11.3, 53000, 56000), (1.37, 11.3, 53000, 56000),
                                                      (17.71, -33.9, 55500, 58800)]):
        ep = np.sort(rng.uniform(lo, hi, 60))
        mjd = np.concatenate([e + rng.uniform(0, 0.9, 3) / 86400.0 for e in ep])
        p = pulsar_from_arrays(f"D{j}", {"RAJ": ra, "DECJ": dec}, mjd.astype(np.longdouble), rng.uniform(0.2, 2.0, mjd.size),
                               flags=[{"f": "A"}] * mjd.size)
        make_ideal(p)
        psrs.append(p)
    b = PulsarBatch(psrs, plan_only=True)
    for i in range(3):
        b.set_white(i, efac=1.1, log10_equad=-6.5)
    b.set_burst_statistic(nside=1)
    pb = b.plan()["burst"]
    assert pb["n_tmpl"] < len(b._burst["templates"])
    assert np.all(pb["seen"][2])                                     # every kept template is seen by the third pulsar
    early = b._burst["templates"][b._burst["templates"][:, 0] < 54500][0]
    b.set_burst_statistic(t0_mjd=[early[0]], f0=[early[1]], Q=[early[2]], nside=1)
    with pytest.raises(ValueError, match=r"M4\(j, s\) at template 0"):
        b.plan()
