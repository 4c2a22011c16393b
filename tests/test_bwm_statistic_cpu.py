"""CPU tests of the burst-with-memory search's host statics (``PulsarBatch.set_bwm_statistic``, ``plan()["bwm"]``) against
the dense oracle (tests/bwm_oracle.py), the bound B <= 1/2 sum_a X^^2, unseen epochs, the default grid, every argument
and plan-time check and the independence of the other statistics' statics.  ``plan_only`` batches: the 3
``partim_small`` pulsars and the 4-pulsar synthetic case of tests/test_optimal_statistic_cpu.py."""
import numpy as np
import pytest

from tests import bwm_oracle as BO
from tests import fe_oracle as EO
from tests.test_fe_statistic_cpu import _live_rows
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# Woodbury (host statics) against dense null-space solves and an explicit P x 2 design matrix per cell (oracle): both
# fp64 evaluations of the same quantity, the bound of the Fp / Fe statics.
TOL = 1e-10
T = 9
CASES = [(src, tm, common) for src in ("small", "synthetic") for tm in (False, True) for common in (None, -14.5)]


def unpack_layout(pb, dtype=np.float64):
    """(sqrt(m) [P, T], antenna [P, S, 2], L2^-1 [T, S, 2, 2]) read back from the kernel layouts of ``plan()["bwm"]``."""
    P, T_, S = pb["sqm"].shape[1], pb["n_t0"], pb["n_sky"]
    sq = np.asarray(pb["sqm"]).transpose(0, 2, 1).reshape(-1, P)[:T_].T
    A = np.asarray(pb["ant"]).copy()
    A[:, 1::2, :] = np.roll(A[:, 1::2, :], -8, axis=-1)
    ant = A.transpose(1, 0, 2).reshape(A.shape[1], -1, 2)[:P, :S]
    lv = np.asarray(pb["linv"]).reshape(pb["linv"].shape[0], -1, 2, 3).transpose(0, 2, 1, 3).reshape(-1, pb["linv"].shape[1], 3)
    Li = np.zeros((T_, S, 2, 2), dtype=dtype)
    Li[..., 0, 0], Li[..., 1, 0], Li[..., 1, 1] = lv[:T_, :S, 0], lv[:T_, :S, 1], lv[:T_, :S, 2]
    return sq.astype(dtype), ant.astype(dtype), Li


def bwm_of_layout(pb, X, dtype=np.float64):
    """B [R, T, S] of whitened amplitudes X [R, P, T] from the kernel layouts of ``plan()["bwm"]``: N2 = sum_a e_a
    sqrt(m_a) X^_a, 1/2 |L2^-1 N2|^2 -- the arithmetic of ptar_bwm_sky, in ``dtype``.  Also returns N2 [R, T, S, 2]."""
    sq, ant, Li = unpack_layout(pb, dtype)
    W = np.asarray(X, dtype=dtype) * sq[None]
    N2 = np.einsum("asp,rat->rtsp", ant, W)
    y = np.einsum("tsij,rtsj->rtsi", Li, N2)
    return 0.5 * np.sum(y * y, axis=-1), N2


def bwm_from_plan(b, pb, rows):
    """(B [R, T, S], X^ [R, P, T]) evaluated in numpy from the plan: X^ from ``Ct`` by ``fp_whitened_basis``."""
    from pta_replicator_b200.engine import fp_whitened_basis
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ fp_whitened_basis(pb, b.toa_off[i], b.ntoa[i])[:, :pb["n_t0"]]
                  for i in range(b.n_psr)], axis=1)
    return bwm_of_layout(pb, X)[0], X


@pytest.mark.parametrize("src,tm,common", CASES)
def test_statics_match_dense_oracle(src, tm, common):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    b.set_bwm_statistic(n_epochs=T, nside=2, log10_A_common=common)
    pb = b.plan()["bwm"]
    assert pb["n_sky"] == 48 and pb["n_t0"] == T and pb["linv"].shape == (5, 64, 6) and pb["ant"].shape == (2, 16, 64)
    models = _models(b) if tm else None
    S = BO.statics(b, pb["t0_mjd"], log10_A_common=common, models=models)
    ant_o = EO.antenna(b, pb["sky"])
    rows = _live_rows(b, 5)
    B, X = bwm_from_plan(b, pb, rows)
    ref, _ = BO.bwm_of_amps(S, ant_o, BO.amps_of_rows(b, S, rows))
    from pta_replicator_b200.engine import fp_whitened_basis
    ct = max(float(np.max(np.abs(fp_whitened_basis(pb, b.toa_off[i], b.ntoa[i])[:, :T] - S["Ct"][i]))
                   / np.max(np.abs(S["Ct"][i]))) for i in range(b.n_psr))
    worst = dict(m=float(np.max(np.abs(pb["m"] - S["m"]) / np.max(S["m"], axis=1, keepdims=True))), Ct=ct,
                 B=float(np.max(np.abs(B - ref)) / np.max(ref)), antenna=float(np.max(np.abs(pb["antenna"] - ant_o))))
    print(f"\n[bwm statics] {src} tm={tm} common={common}: seen {int(pb['seen'].sum())}/{pb['seen'].size}, "
          + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert max(worst.values()) < TOL, worst
    assert np.array_equal(pb["seen"], S["seen"])
    # B is the projection of 1/2 sum_a X^^2 onto a 2-dimensional subspace
    assert np.all(B <= 0.5 * np.sum(X * X, axis=1)[:, :, None] * (1 + 1e-12))


def test_invariant_on_every_cell():
    b = _batch(_synthetic(), tm=True)
    b.set_bwm_statistic(t0_mjd=np.linspace(53300.0, 58400.0, 40), nside=4, log10_A_common=-14.5)
    pb = b.plan()["bwm"]
    B, X = bwm_from_plan(b, pb, _live_rows(b, 16, seed=7))
    ratio = float(np.max(B / (0.5 * np.sum(X * X, axis=1))[:, :, None]))
    print(f"\n[bwm] max B / (1/2 sum X^2) over {B.size} cells: {ratio:.6f}")
    assert ratio <= 1 + 1e-12
    assert pb["M2"].shape == (40, 192, 2, 2)


def test_unseen_epochs_and_padding():
    """A ramp starting before a pulsar's first TOA is a line on every TOA: an offset + F0 timing model absorbs it, so the
    epoch is unseen (zero column, m = 0); without a timing model it is seen.  After the last TOA the ramp is zero."""
    psrs = _synthetic()
    first = [float(np.min(p.toas.get_mjds().value)) for p in psrs]
    last = [float(np.max(p.toas.get_mjds().value)) for p in psrs]
    j = int(np.argmax(first))                                 # the pulsar that starts last: the others see t_before
    k = int(np.argmin(last))                                  # the pulsar that ends first: the others see t_after
    t_before, t_after = first[j] - 20.0, last[k] + 20.0
    t0 = np.array([t_before, 55000.0, 56000.5, t_after, 57000.0])
    for tm in (True, False):
        b = _batch(psrs, tm=tm)
        b.set_bwm_statistic(t0_mjd=t0, nside=1)
        pb = b.plan()["bwm"]
        assert bool(pb["seen"][j, 0]) is (not tm), tm
        assert not pb["seen"][k, 3] and pb["m"][k, 3] == 0.0
        assert np.sum(pb["seen"]) == 4 * 5 - 1 - int(tm)
        from pta_replicator_b200.engine import fp_whitened_basis
        for i in range(b.n_psr):
            W = fp_whitened_basis(pb, b.toa_off[i], b.ntoa[i])
            assert W.shape[1] == 6 and np.all(W[:, 5] == 0)  # T = 5 padded to 6 columns
            assert np.all(W[:, :5][:, ~pb["seen"][i]] == 0) and np.all(np.any(W[:, :5][:, pb["seen"][i]] != 0, axis=0))
        sq, _, _ = unpack_layout(pb)
        assert np.array_equal(sq, np.sqrt(pb["m"]))
        assert np.all(pb["sqm"][2, :, 1] == 0) and np.all(pb["linv"][2, :, 3:] == 0)     # the absent sixth epoch
        assert np.all(pb["linv"][:, 12:] == 0) and np.all(pb["ant"][:, b.n_psr:, :] == 0)  # past S and P
        un = pb["Ct"].copy()                                  # columns past 2 ceil(T / 2) of every TOA
        un[:, 1::2, :] = np.roll(un[:, 1::2, :], -8, axis=-1)
        assert pb["Ct"].shape[0] == 1 and np.all(un[0][:, 6:] == 0)


def test_default_grid():
    b = _batch(_synthetic())
    b.set_bwm_statistic(n_epochs=7, nside=1)
    lo = min(float(m.min()) for m in b.mjd)
    hi = max(float(m.max()) for m in b.mjd)
    t0 = b._bwm["t0_mjd"]
    assert np.allclose(t0, lo + (np.arange(7) + 0.5) * (hi - lo) / 7, rtol=0, atol=1e-9)
    from pta_replicator_b200.engine import healpix_ring_centres
    assert np.array_equal(b._bwm["sky"], healpix_ring_centres(1))
    assert np.array_equal(b.plan()["bwm"]["t0_mjd"], t0) and b.bwm_setup_s is not None


def test_value_errors():
    from pta_replicator_b200 import orf
    from pta_replicator_b200.engine import PulsarBatch
    from tests import reduction_reference as RR
    psrs = _synthetic()
    b = _batch(psrs)
    for bad, msg in (([], "empty"), ([55000.0, np.nan], "finite"), ([55000.0, np.inf], "finite"),
                     ([55000.0, 55000.0], "duplicates"), (np.linspace(53000, 58000, 513), "at most 512")):
        with pytest.raises(ValueError, match=msg):
            b.set_bwm_statistic(t0_mjd=bad)
    for bad in (0, -3, 513, 2.5, True):
        with pytest.raises(ValueError, match="n_epochs"):
            b.set_bwm_statistic(n_epochs=bad)
    for bad in (0, 3, 64, 2.0, True):
        with pytest.raises(ValueError, match="nside"):
            b.set_bwm_statistic(nside=bad)
    for bad, msg in ((np.zeros((0, 2)), "empty"), (np.array([[1.0, np.nan]]), "finite"), (np.zeros((3, 3)), r"\[S, 2\]"),
                     (np.ones((12289, 2)), "at most 12288")):
        with pytest.raises(ValueError, match=msg):
            b.set_bwm_statistic(sky=bad)
    for kw, msg in ((dict(log10_A_common=np.nan), "log10_A_common"), (dict(gamma_common=np.inf), "gamma_common"),
                    (dict(components_common=0), "components_common")):
        with pytest.raises(ValueError, match=msg):
            b.set_bwm_statistic(**kw)
    assert b._bwm is None                                     # nothing was registered by a failed call
    with pytest.raises(ValueError, match="at least 2 pulsars"):
        _batch(psrs[:1]).set_bwm_statistic()
    big = PulsarBatch(RR.edge_pulsars((5,) * 129, seed=2), plan_only=True)
    with pytest.raises(ValueError, match="at most 128 pulsars"):
        big.set_bwm_statistic()
    # plan time: missing white noise
    nw = _batch(psrs, white=False)
    nw.set_bwm_statistic(n_epochs=4, nside=1)
    with pytest.raises(ValueError, match="white noise"):
        nw.plan()
    # a pulsar that sees no epoch: every epoch after its last TOA
    last = [float(np.max(p.toas.get_mjds().value)) for p in psrs]
    k = int(np.argmin(last))
    late = _batch(psrs)
    late.set_bwm_statistic(t0_mjd=[last[k] + 5.0, last[k] + 10.0], nside=1)
    with pytest.raises(ValueError, match=f"pulsar {k} \\({psrs[k].name}\\) sees no burst epoch"):
        late.plan()
    # staggered spans: an epoch only one pulsar sees
    two = _batch(psrs[:2])
    l2 = [float(np.max(p.toas.get_mjds().value)) for p in psrs[:2]]
    t_one = min(l2) + 0.5 * (max(l2) - min(l2))
    two.set_bwm_statistic(t0_mjd=[55000.0, t_one], nside=1)
    with pytest.raises(ValueError, match=r"epoch index 1\), sky point 0 .* not safely positive definite.*pass t0_mjd"):
        two.plan()
    # two pulsars and a sky point on one of them: one antenna pattern, M2 has rank 1
    locs = orf.psrlocs_from_pulsars(two.psrs)
    two.set_bwm_statistic(t0_mjd=[55000.0], sky=np.array([[1.0, 2.0], [np.pi / 2 - locs[0, 1], locs[0, 0]]]))
    with pytest.raises(ValueError, match=r"epoch index 0\), sky point 1 .* not safely positive definite"):
        two.plan()


def test_registration_leaves_other_statistics_unchanged():
    b = _batch(_synthetic(), tm=True)
    b.set_optimal_statistic(components=4)
    b.set_fp_statistic(n_freqs=5, log10_A_common=-14.5)
    b.set_fe_statistic(nside=1)
    b.set_curn_likelihood(log10_A=np.linspace(-16, -13, 4), gamma=[3.0, 13 / 3], components=4)
    b.set_red_noise_likelihood(log10_A=np.linspace(-16, -13, 4), gamma=[3.0, 13 / 3], components=4)
    plain = b.plan()
    assert plain["bwm"] is None and b.bwm_setup_s is None
    b.set_bwm_statistic(n_epochs=6, nside=1, log10_A_common=-14.5)
    both = b.plan()
    for key in ("fp", "fe", "os", "curn", "rn"):
        for k, v in plain[key].items():
            if isinstance(v, np.ndarray):
                assert np.array_equal(v, both[key][k]), (key, k)
    assert both["bwm"]["n_t0"] == 6 and both["bwm"]["setup_s"] == b.bwm_setup_s


def test_sky_model_checks_refuse_before_any_launch():
    """``ptar_fe_sky`` / ``ptar_fe_combine`` and ``ptar_bwm_sky`` / ``ptar_bwm_combine`` share one check of the sky grid
    (the model arrays, n_psr and kp, n_sky and n_sb, the 16-byte alignment of the staged arrays), and each checks its
    frequency or epoch count; every call below refuses its model before anything reaches a device."""
    import ctypes as C

    from pta_replicator_b200 import _cabi
    L = _cabi.lib()
    buf = (C.c_double * 64)()
    p = (C.addressof(buf) + 15) & ~15                     # 16-byte aligned, never read: every call stops at its checks
    sky = dict(n_psr=3, kp=16, n_sky=40, n_sb=2, ant=p, linv=p)

    def fe(**kw):
        return _cabi.FeModel(**{**sky, "n_freq": 4, "Lf": p, **kw})

    def bw(**kw):
        return _cabi.BwmModel(**{**sky, "n_t0": 5, "sqm": p, "seen": p, "antenna": p, **kw})

    shared = [(dict(ant=None), "model arrays missing"), (dict(linv=None), "model arrays missing"),
              (dict(n_psr=0), "1 <= n_psr <= 128"), (dict(n_psr=129, kp=144), "1 <= n_psr <= 128"),
              (dict(kp=32), "kp = n_psr rounded up"), (dict(n_sky=0, n_sb=0), "1 <= n_sky <= 12288"),
              (dict(n_sb=1), "n_sb = ceil(n_sky / 32)"), (dict(n_sky=12289, n_sb=385), "1 <= n_sky <= 12288")]
    fe_own = [(dict(Lf=None), "model arrays missing"), (dict(n_freq=0), "1 <= n_freq <= 256"),
              (dict(n_freq=257), "1 <= n_freq <= 256"), (dict(ant=p + 8), ": ant and linv must be 16-byte aligned"),
              (dict(linv=p + 8), ": ant and linv must be 16-byte aligned")]
    bw_own = [(dict(sqm=None), "model arrays missing"), (dict(seen=None), "model arrays missing"),
              (dict(antenna=None), "model arrays missing"), (dict(n_t0=0), "1 <= n_t0 <= 512"),
              (dict(n_t0=513), "1 <= n_t0 <= 512"), (dict(sqm=p + 8), ": sqm, ant and linv must be 16-byte aligned"),
              (dict(ant=p + 8), ": sqm, ant and linv must be 16-byte aligned"),
              (dict(linv=p + 8), ": sqm, ant and linv must be 16-byte aligned")]
    calls = {"ptar_fe_sky": (fe, fe_own, lambda m: L.ptar_fe_sky(p, 4, C.byref(m), p, p, None, None)),
             "ptar_fe_combine": (fe, fe_own, lambda m: L.ptar_fe_combine(p, p, 4, C.byref(m), p, p, p, None)),
             "ptar_bwm_sky": (bw, bw_own, lambda m: L.ptar_bwm_sky(p, 4, C.byref(m), p, p, None, None)),
             "ptar_bwm_combine": (bw, bw_own, lambda m: L.ptar_bwm_combine(p, p, p, 4, C.byref(m), *([p] * 10), None))}
    for name, (model, own, call) in calls.items():
        for kw, msg in shared + own:
            assert call(model(**kw)) == -2, (name, kw)
            err = L.ptar_last_error().decode()
            assert err.startswith(name + ": ") and msg in err, (name, kw, err)
