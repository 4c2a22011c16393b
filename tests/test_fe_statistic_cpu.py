"""CPU tests of the Fe-statistic's host statics (``PulsarBatch.set_fe_statistic``, ``plan()["fe"]``) against the dense
oracle (tests/fe_oracle.py), the bound Fe <= Fp, the HEALPix grid, the antenna pattern at a pulsar's own position and
every argument check.  ``plan_only`` batches: the 3 ``partim_small`` pulsars and the 4-pulsar synthetic case of
tests/test_optimal_statistic_cpu.py."""
import numpy as np
import pytest

from tests import fe_oracle as EO
from tests import fp_oracle as FO
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# Woodbury + closed-form 2 x 2 Cholesky + inverse Cholesky of M4 (host statics) against dense solves with the explicit
# 2P x 4 design matrix (oracle): both are fp64 evaluations of the same quantity; the Fp statics' bound.
TOL = 1e-10
NF = 12
CASES = [(src, tm, common) for src in ("small", "synthetic") for tm in (False, True) for common in (None, -14.5)]


def _live_rows(b, R, seed=1):
    rows = np.random.default_rng(seed).standard_normal((R, b.ld)) * 1e-6
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    rows[:, ~live] = 0
    return rows


def fe_of_layout(Lf, ant_k, linv, P, S, X, dtype=np.float64):
    """Fe [R, Nf, S] of whitened amplitudes X [R, P, Nf, 2] from the kernel layouts of ``plan()["fe"]`` (``Lf``, ``ant``
    with the odd-pulsar rotation undone, ``linv``): N = L X^, N4 = sum_a e_a (x) N_a, 1/2 |L4^-1 N4|^2 -- the arithmetic of
    ptar_fe_sky, in ``dtype``.  Also returns the antenna patterns [P, S, 2] read back from the layout."""
    X = np.asarray(X, dtype=dtype)
    A = np.asarray(ant_k).copy()
    A[:, 1::2, :] = np.roll(A[:, 1::2, :], -8, axis=-1)
    ant = A.transpose(1, 0, 2).reshape(A.shape[1], -1, 2)[:P, :S]          # [P, S, 2]
    L = np.asarray(Lf, dtype=dtype).transpose(1, 0, 2)[None]              # [1, P, Nf, 3]
    N = np.stack([L[..., 0] * X[..., 0], L[..., 1] * X[..., 0] + L[..., 2] * X[..., 1]], axis=-1)
    R, Nf = X.shape[0], X.shape[2]
    N4 = np.einsum("asp,rafc->rfspc", ant.astype(dtype), N).reshape(R, Nf, S, 4)
    Li = np.zeros((Nf, S, 4, 4), dtype=dtype)
    Li[..., np.tril_indices(4)[0], np.tril_indices(4)[1]] = np.asarray(linv)[:, :S]
    y = np.einsum("fsij,rfsj->rfsi", Li, N4)
    return 0.5 * np.sum(y * y, axis=-1), ant


def fe_from_plan(b, pl, rows):
    """Fe [R, Nf, S] and Fp [R, Nf] evaluated in numpy from the plan: X^ from ``Ct``, then ``fe_of_layout``."""
    from pta_replicator_b200.engine import fp_whitened_basis
    pf, pe = pl["fp"], pl["fe"]
    P, Nf, R = b.n_psr, pf["n_freq"], rows.shape[0]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ fp_whitened_basis(pf, b.toa_off[i], b.ntoa[i])
                  for i in range(P)], axis=1).reshape(R, P, Nf, 2)
    fe, ant = fe_of_layout(pe["Lf"], pe["ant"], pe["linv"], P, pe["n_sky"], X)
    return fe, 0.5 * np.sum(X * X, axis=(1, 3)), ant


@pytest.mark.parametrize("src,tm,common", CASES)
def test_statics_match_dense_oracle(src, tm, common):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    b.set_fp_statistic(n_freqs=NF, log10_A_common=common)
    b.set_fe_statistic(nside=2)
    pl = b.plan()
    pe = pl["fe"]
    assert pe["n_sky"] == 48 and pe["linv"].shape == (NF, 64, 10) and pe["ant"].shape == (2, 16, 64)
    S = FO.statics(b, pl["fp"]["freqs"], log10_A_common=common, models=_models(b) if tm else None)
    ant_o = EO.antenna(b, pe["sky"])
    rows = _live_rows(b, 5)
    fe, fp, ant = fe_from_plan(b, pl, rows)
    ref = EO.fe_of_rows(b, S, ant_o, rows)
    worst = dict(antenna=float(np.max(np.abs(ant - ant_o))),
                 Fe=float(np.max(np.abs(fe - ref)) / np.max(ref)),
                 Fe_cell=float(np.max(np.abs(fe - ref) / ref)))
    print(f"\n[fe statics] {src} tm={tm} common={common}: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert max(worst.values()) < TOL, worst
    # Fe is the projection of 2Fp onto a 4-dimensional subspace
    assert np.all(fe <= fp[:, :, None] * (1 + 1e-12))
    # padding carries no weight
    assert np.all(pe["linv"][:, 48:] == 0) and np.all(pe["ant"][:, b.n_psr:, :] == 0)


def test_fe_never_exceeds_fp_on_every_cell():
    b = _batch(_synthetic(), tm=True)
    b.set_fp_statistic(n_freqs=40, log10_A_common=-14.5)
    b.set_fe_statistic(nside=4)
    pl = b.plan()
    fe, fp, _ = fe_from_plan(b, pl, _live_rows(b, 16, seed=7))
    ratio = float(np.max(fe / fp[:, :, None]))
    print(f"\n[fe] max Fe / Fp over {fe.size} cells: {ratio:.6f}")
    assert ratio <= 1 + 1e-12
    assert pl["fe"]["M4"].shape == (40, 192, 4, 4)


def test_healpix_ring_centres():
    from pta_replicator_b200.engine import healpix_ring_centres
    for nside in (1, 2, 4, 8, 16, 32):
        c = healpix_ring_centres(nside)
        assert c.shape == (12 * nside * nside, 2)
        z = np.cos(c[:, 0])
        assert np.allclose(np.sort(z), np.sort(-z), rtol=0, atol=1e-15)          # symmetric about the equator
        v = np.stack([np.sin(c[:, 0]) * np.cos(c[:, 1]), np.sin(c[:, 0]) * np.sin(c[:, 1]), z], axis=1)
        assert np.max(np.abs(v.mean(axis=0))) < 1e-15
        assert np.all((c[:, 1] >= 0) & (c[:, 1] < 2 * np.pi)) and np.all(np.diff(z) <= 1e-15)   # rings north to south
        assert len(np.unique(np.round(v, 12), axis=0)) == len(c)
    c = healpix_ring_centres(1)
    th = np.r_[[np.arccos(2 / 3)] * 4, [np.pi / 2] * 4, [np.arccos(-2 / 3)] * 4]
    ph = np.r_[np.arange(4) * np.pi / 2 + np.pi / 4, np.arange(4) * np.pi / 2, np.arange(4) * np.pi / 2 + np.pi / 4]
    assert np.allclose(c[:, 0], th, rtol=0, atol=1e-15) and np.allclose(c[:, 1], ph, rtol=0, atol=1e-15)
    # nside 2: ring z = 1 - 1/12, 1 - 4/12 (caps), then the belt at (2 - i) / 3
    z = np.cos(healpix_ring_centres(2)[:, 0])
    assert np.allclose(z[:4], 11 / 12) and np.allclose(z[4:12], 2 / 3) and np.allclose(z[12:20], 1 / 3)
    assert np.allclose(z[-4:], -11 / 12)


def test_zero_antenna_at_a_pulsars_own_position():
    from pta_replicator_b200 import orf
    b = _batch(_synthetic())
    b.set_fp_statistic(n_freqs=3)
    locs = orf.psrlocs_from_pulsars(b.psrs)
    sky = np.array([[np.pi / 2 - locs[1, 1], locs[1, 0]], [1.0, 2.0]])
    b.set_fe_statistic(sky=sky)
    pe = b.plan()["fe"]
    assert np.array_equal(pe["antenna"][1, 0], [0.0, 0.0])
    assert np.all(np.abs(pe["antenna"][[0, 2, 3], 0]).sum(axis=1) > 0) and np.all(np.abs(pe["antenna"][:, 1]).sum(axis=1) > 0)
    # the oracle's own evaluation agrees
    assert np.allclose(EO.antenna(b, sky), pe["antenna"], rtol=0, atol=1e-13)


def test_registration_follows_the_fp_statistic():
    b = _batch(_synthetic())
    b.set_fp_statistic(n_freqs=5)
    plain = b.plan()
    assert plain["fe"] is None and b.fe_setup_s is None
    b.set_fe_statistic(nside=1)
    both = b.plan()
    for k, v in plain["fp"].items():                          # the Fp statics do not depend on the sky grid
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, both["fp"][k]), k
    assert both["fe"]["n_sky"] == 12 and b.fe_setup_s is not None and both["fe"]["setup_s"] == b.fe_setup_s
    assert np.array_equal(both["fe"]["Lf"][:, :, 0], np.sqrt(both["fp"]["M"][:, :, 0, 0]).T)
    b.set_fp_statistic(n_freqs=5)                             # re-registering Fp clears the sky grid
    assert b._fe is None and b.plan()["fe"] is None


def test_value_errors():
    psrs = _synthetic()
    b = _batch(psrs)
    with pytest.raises(ValueError, match="set_fp_statistic"):
        b.set_fe_statistic()
    b.set_fp_statistic(n_freqs=4)
    for bad in (0, 3, 64, 2.0, True, -8):
        with pytest.raises(ValueError, match="nside"):
            b.set_fe_statistic(nside=bad)
    for bad, msg in ((np.zeros((0, 2)), "empty"), (np.array([[1.0, np.nan]]), "finite"), (np.array([[np.inf, 1.0]]), "finite"),
                     (np.zeros((3, 3)), r"\[S, 2\]"), (np.zeros(4), r"\[S, 2\]"), (np.ones((12289, 2)), "at most 12288")):
        with pytest.raises(ValueError, match=msg):
            b.set_fe_statistic(sky=bad)
    assert b._fe is None                                      # nothing was registered by a failed call
    # more pulsars than the kernel's shared-memory tile holds
    from tests import reduction_reference as RR
    from pta_replicator_b200.engine import PulsarBatch
    big = PulsarBatch(RR.edge_pulsars((5,) * 129, seed=2), plan_only=True)
    big._fp = dict(b._fp)
    with pytest.raises(ValueError, match="at most 128 pulsars"):
        big.set_fe_statistic()
    # two pulsars and a sky point on one of them: only one antenna pattern, M4 has rank 2
    from pta_replicator_b200 import orf
    two = _batch(psrs[:2])
    two.set_fp_statistic(n_freqs=4)
    locs = orf.psrlocs_from_pulsars(two.psrs)
    two.set_fe_statistic(sky=np.array([[1.0, 2.0], [np.pi / 2 - locs[0, 1], locs[0, 0]]]))
    with pytest.raises(ValueError, match=r"frequency index 0\), sky point 1 .* not safely positive definite"):
        two.plan()
    # one pulsar: M4 is singular everywhere
    one = _batch(psrs[:1])
    one.set_fp_statistic(n_freqs=2)
    one.set_fe_statistic(nside=1)
    with pytest.raises(ValueError, match="not safely positive definite"):
        one.plan()
