"""Chromatic noise (DM and scattering Gaussian processes) on the host, without a device: the recipe API and its
refusals, the Taylor window over every process, the DM timing-model columns, the noise dictionary keys, and
``_pinv_apply`` with chromatic blocks against the extended-precision dense P^-1 of tests/statics_reference.py."""
import math

import numpy as np
import pytest

from tests import statics_reference as SR


def chrom_pulsars(ntoas, seed=0, single=(), nofreq=()):
    """Pulsars of epochs with 1-8 sub-band TOAs < 1 s apart, spread over 700-1900 MHz; pulsars in ``single`` observe at
    one frequency only, pulsars in ``nofreq`` carry a zero frequency on their first TOA."""
    from pta_replicator_b200.simulate import make_ideal, pulsar_from_arrays
    rng = np.random.default_rng(seed)
    out = []
    for j, n in enumerate(ntoas):
        sub = []
        while sum(sub) < n:
            sub.append(int(min(rng.integers(1, 9), n - sum(sub))))
        ep = np.sort(rng.uniform(53000.0, 58800.0, len(sub)))
        mjd = np.concatenate([e + np.sort(rng.uniform(0, 0.9, k)) / 86400.0 for e, k in zip(ep, sub)])
        nu = np.concatenate([np.linspace(700.0, 1900.0, k) if k > 1 else [1400.0] for k in sub])
        if j in single:
            nu = np.full(n, 820.0)
        if j in nofreq:
            nu[0] = 0.0
        ra, dec = rng.uniform(0, 24), math.degrees(math.asin(rng.uniform(-1, 1)))
        p = pulsar_from_arrays(f"C{j:03d}", {"RAJ": float(ra), "DECJ": float(dec)}, mjd.astype(np.longdouble),
                               rng.uniform(0.3, 3.0, n), freq=nu)
        make_ideal(p)
        out.append(p)
    return out


def _batch(ntoas=(40, 25, 60), **kw):
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(chrom_pulsars(ntoas, **{k: kw.pop(k) for k in ("single", "nofreq") if k in kw}), plan_only=True, **kw)
    for i in range(b.n_psr):
        b.set_white(i, efac=1.1)
    return b


def test_freq_is_read_in_engine_order():
    b = _batch()
    for i, p in enumerate(b.psrs):
        assert np.array_equal(b.freq[i], np.asarray(p.toas.table["freq"])[b.order[i]])
        assert np.array_equal(p.toas.table["freq"], p.toas.freq)


def test_refusals():
    b = _batch(nofreq=(1,))
    with pytest.raises(ValueError, match="radio frequency"):
        b.set_dm_noise(1, -13.0, 2.0)
    with pytest.raises(ValueError, match="finite idx"):
        b.set_chromatic_noise(0, -13.0, 2.0, idx=np.nan)
    with pytest.raises(ValueError, match="fref"):
        b.set_dm_noise(0, -13.0, 2.0, fref=np.inf)
    b.set_dm_noise(0, -13.0, 2.0, components=10)
    with pytest.raises(ValueError, match="same number of components"):
        b.set_dm_noise(2, -13.0, 2.0, components=12)
    b.set_chromatic_noise(2, -13.0, 2.0, components=12)   # the other slot has its own count
    with pytest.raises(ValueError, match="dm columns"):
        b.set_timing_model(1, dm=2)


def test_subset_and_weights():
    b = _batch()
    b.set_dm_noise(0, -13.0, 2.5, components=8, fref=1000.0)
    b.set_chromatic_noise(2, -13.5, 3.0, idx=4.4, components=5)
    pl = b.plan()
    dm, ch = pl["chrom"]
    assert dm["J"] == 16 and ch["J"] == 10
    assert list(dm["on"]) == [1, 0, 0] and list(ch["on"]) == [0, 0, 1]
    s0, s2 = b.toa_off[0], b.toa_off[2]
    assert np.array_equal(dm["weight"][s0:s0 + b.ntoa[0]], (1000.0 / b.freq[0]) ** 2)
    assert np.array_equal(ch["weight"][s2:s2 + b.ntoa[2]], (1400.0 / b.freq[2]) ** 4.4)
    assert not np.any(dm["weight"][b.toa_off[1]:])
    assert np.all(dm["scale"][1:] == 0) and np.all(ch["freqs"][:2] == 0)
    # one basis row per epoch of every tile of the pulsars that carry the slot
    tiles = pl["tiles"]
    assert len(dm["frow_t"]) == int(tiles[tiles[:, 5] == 0, 4].sum())


def test_prior_is_set_reds():
    b = _batch()
    b.set_red(0, -13.2, 3.1, components=7)
    b.set_dm_noise(0, -13.2, 3.1, components=7)
    assert np.array_equal(b._red["scale"][0], b._chrom[0]["scale"][0])
    assert np.array_equal(b._red["f"][0], b._chrom[0]["f"][0])


def test_taylor_window_is_the_minimum_over_processes():
    b = _batch(ntoas=(300,))
    base = _batch(ntoas=(300,))
    for x in (b, base):
        x.set_red(0, -14.0, 4.0, components=5)
    ref = base.plan()
    b.set_dm_noise(0, -13.0, 1.0, components=30)    # flat, many components: a much shorter window
    m2, m3 = b._taylor_moments(0)
    r2, r3 = base._taylor_moments(0)
    assert m2 > r2 and m3 > r3
    c = b._chrom[0]
    w = 2 * np.pi * c["f"][0]
    sk = c["scale"][0][0::2]
    assert m3 == pytest.approx(4 * np.sum(sk * w ** 3) / np.sqrt(np.sum(sk * sk)), rel=1e-15)
    pl = b.plan()
    assert pl["n_epochs"] >= ref["n_epochs"]
    # every epoch respects the chromatic window
    tol = b.rn_taylor_tol
    dmax = (6 * tol / m3) ** (1.0 / 3.0)
    ep, first = b._epochs_for(0, 0.0)[:2]
    t = b.t_tdb[0]
    assert np.all(t - t[first][ep] <= dmax * (1 + 1e-12))


def _red_only_moments(b, i):
    """The red-noise-only Taylor moments (the rule without chromatic slots), written out independently."""
    w = 2 * np.pi * np.asarray(b._red["f"][i], dtype=float)
    sk = np.asarray(b._red["scale"][i], dtype=float)[0::2]
    nrm = float(np.sqrt(np.sum(sk * sk)))
    return (0.0, 0.0) if nrm == 0.0 else (4.0 * float(np.sum(sk * w**2)) / nrm, 4.0 * float(np.sum(sk * w**3)) / nrm)


def _epochs_by_rule(b, i, m3):
    """Epoch index per TOA from the documented rule: cuts at ECORR-bucket changes and wherever the run from the epoch's
    first TOA would pass the window (6 tol / m3)^(1/3); the tile cut does not matter here."""
    t, bucket = b.t_tdb[i], b._ecorr[i][0]
    dmax = np.inf if m3 <= 0 else (6 * b.rn_taylor_tol / m3) ** (1.0 / 3.0)
    ep = np.zeros(len(t), dtype=np.int64)
    start = 0
    for k in range(1, len(t)):
        if bucket[k] != bucket[k - 1] or t[k] - t[start] > dmax:
            start = k
            ep[k] = ep[k - 1] + 1
        else:
            ep[k] = ep[k - 1]
    return ep


def test_without_chromatic_noise_the_plan_follows_the_red_noise_rule():
    """No chromatic slot: the Taylor moments are the red-noise-only formula bit for bit, the epochs follow that
    formula's window, and the plan carries no chromatic statics."""
    from tests import generator_reference as GR
    b = GR.gen_batch(plan_only=True, ntoas=(1, 5, 300, 1100, (64, 1)), dense=(), red=10)
    pl = b.plan()
    assert pl["chrom"] is None
    for i in range(b.n_psr):
        m = _red_only_moments(b, i)
        assert b._taylor_moments(i) == m
        ep = b._epochs_for(i, 0.0)[0]
        assert np.array_equal(ep, _epochs_by_rule(b, i, m[1])), i


def test_chromatic_plan_leaves_other_statics_alone_when_windows_agree():
    # a chromatic process no faster than the red noise leaves the epochs as they are
    a, b = _batch(), _batch()
    for x in (a, b):
        for i in range(x.n_psr):
            x.set_red(i, -13.0, 4.0, components=10)
    b.set_dm_noise(1, -15.0, 6.0, components=3)
    pa, pb = a.plan(), b.plan()
    for k in ("tiles", "dtau", "eloc", "ep_tref"):
        assert np.array_equal(pa[k], pb[k]), k


def test_dm_timing_model_columns():
    b = _batch()
    b.set_timing_model(0, poly=2, dm=2)
    m = b._tm[0]
    assert m["k"] == 6
    t = b.t_tdb[0]
    x = (t - 0.5 * (t.max() + t.min())) / (0.5 * (t.max() - t.min()))
    w = (1400.0 / b.freq[0]) ** 2
    M = np.stack([x ** 0, x, x ** 2, w, w * x, w * x ** 2], axis=1) * m["sqrtw"][:, None]
    # Q spans the whitened columns
    assert np.allclose(m["Q"] @ (m["Q"].T @ M), M, rtol=0, atol=1e-12 * np.abs(M).max())
    b.set_timing_model(1, poly=None, dm=0)
    assert b._tm[1]["k"] == 1
    b.set_timing_model(2, poly=2)
    assert b._tm[2]["k"] == 3
    # a single-frequency pulsar: DM is an offset, the model is rank-deficient
    s = _batch(ntoas=(30,), single=(0,))
    with pytest.raises(ValueError, match="rank-deficient"):
        s.set_timing_model(0, poly=2, dm=1)


def test_noise_dict_keys():
    from pta_replicator_b200 import noise_dict
    d = {"J0_dm_gp_log10_A": -13.5, "J0_dm_gp_gamma": 2.5, "J0_chrom_gp_log10_A": -14.0, "J0_chrom_gp_gamma": 3.0,
         "J0_red_noise_log10_A": -14.2, "J0_red_noise_gamma": 4.1, "J0_X_efac": 1.1,
         "J1_chrom_gp_log10_A": -14.0, "J1_chrom_gp_gamma": 3.0, "J1_chrom_gp_idx": 4.4}
    p0 = noise_dict.per_pulsar(d, "J0")
    assert (p0["dm_log10_A"], p0["dm_gamma"], p0["chrom_log10_A"], p0["chrom_gamma"], p0["chrom_idx"]) == \
        (-13.5, 2.5, -14.0, 3.0, 4.0)
    assert p0["rn_log10_A"] == -14.2 and p0["backends"] == ["X"]
    p1 = noise_dict.per_pulsar(d, "J1")
    assert p1["dm_log10_A"] is None and p1["dm_gamma"] is None and p1["chrom_idx"] == 4.4
    p2 = noise_dict.per_pulsar(d, "J2")
    assert all(p2[k] is None for k in ("dm_log10_A", "dm_gamma", "chrom_log10_A", "chrom_gamma", "chrom_idx"))


def test_ng15_dictionary_parses_as_before():
    from pta_replicator_b200 import noise_dict
    nd = noise_dict.load_noise_dict()
    names = noise_dict.pulsar_names(nd, require_red=False)
    assert names
    for n in names:
        p = noise_dict.per_pulsar(nd, n)
        assert all(p[k] is None for k in ("dm_log10_A", "dm_gamma", "chrom_log10_A", "chrom_gamma", "chrom_idx"))
        assert set(p) == {"backends", "efac", "log10_equad", "log10_ecorr", "rn_log10_A", "rn_gamma", "dm_log10_A",
                          "dm_gamma", "chrom_log10_A", "chrom_gamma", "chrom_idx"}


# ------------------------------------------------------------------ P^-1 with chromatic blocks
@pytest.mark.parametrize("case", ["all", "single_freq", "chrom_no_red", "dm_only"])
def test_pinv_apply_with_chromatic_blocks(case):
    b = _batch(ntoas=(90, 70, 50), single=(1,) if case == "single_freq" else ())
    tm = dict(poly=2, dm=1) if case == "all" else dict(poly=2)
    for i in range(b.n_psr):
        b.set_ecorr(i, -6.5, coarsegrain=1.0 / 86400.0)
        if case != "chrom_no_red" and case != "dm_only":
            b.set_red(i, -13.6, 3.8, components=6)
        b.set_dm_noise(i, -13.2, 2.2, components=8)
        if case != "dm_only":
            b.set_chromatic_noise(i, -13.8, 3.5, idx=4.0, components=5)
        b.set_timing_model(i, poly=tm["poly"], dm=tm.get("dm"))
    b._ref_chrom = {(slot, i): rec for i in range(b.n_psr) for slot, rec in ((0, (2.0, 1400.0)), (1, (4.0, 1400.0)))}
    for i in range(b.n_psr):
        F = SR.basis(b.t_tdb[i], np.arange(1, 4) / 3e8)
        d = b._white_variances("test")[i]
        got = b._pinv_apply(i, d, F)
        ref = np.asarray(SR.dense_pinv(b, i, F, tm=tm), dtype=float)
        scale = np.abs(ref).max(axis=0)
        assert np.all(np.abs(got - ref) <= 1e-8 * scale), (case, i, float(np.max(np.abs(got - ref) / scale)))


def test_own_red_false_keeps_chromatic_noise():
    b = _batch()
    b.set_red(0, -13.5, 4.0, components=5)
    b.set_red(1, -13.5, 4.0, components=5)
    b.set_red(2, -13.5, 4.0, components=5)
    b.set_dm_noise(0, -13.0, 2.0, components=6)
    blocks, iprior = b._woodbury_blocks(0, own_red=False)
    assert len(blocks) == 1 and blocks[0].shape[1] == 12
    blocks, iprior = b._woodbury_blocks(0)
    assert [x.shape[1] for x in blocks] == [10, 12]
