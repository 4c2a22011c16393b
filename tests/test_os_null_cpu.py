"""CPU tests of the null-distribution statics of the optimal statistic (``PulsarBatch.set_os_null``,
``plan()["os_null"]``): the plan's V and D_s applied in numpy against the dense oracle (tests/os_oracle.py,
tests/os_null_oracle.py) computed from scratch with a literally phase-shifted GW basis or with the closed-form templates
at the scrambled positions, the scramble acceptance rule and seeding, and the argument checks.  ``plan_only`` batches:
the 3 ``partim_small`` pulsars and the 4-pulsar synthetic case of test_optimal_statistic_cpu.py."""
import numpy as np
import pytest

from tests import os_null_oracle as NO
from tests import os_oracle as OO
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

NCOL = 8
K = 10


def u_of_x(x, pairs, method):
    """The GEMM's left operand U [R, kd] from x = X phi~^{1/2} [R, P, 2K], in the order of ptar_os_null."""
    xa, xb = x[:, pairs[:, 0]], x[:, pairs[:, 1]]                          # [R, n_pairs, 2K]
    if method == "sky_scramble":
        return np.einsum("rqj,rqj->rq", xa, xb)
    sa, ca, sb, cb = xa[..., 0::2], xa[..., 1::2], xb[..., 0::2], xb[..., 1::2]
    U = np.stack([sa * sb + ca * cb, ca * sb - sa * cb], axis=-1)             # [R, n_pairs, K, 2]
    return U.reshape(len(x), -1)


def _setup(src, tm, method, template="hd", seed=5, match=0.1):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    orfs = ("hd", "monopole", "dipole") if b.n_psr > 3 else ("hd", "monopole")
    b.set_optimal_statistic(components=K, orfs=orfs)
    b.set_os_null(method, n=NCOL, seed=seed, template=template, match=match)
    pl = b.plan()
    models = _models(b) if tm else None
    S0 = OO.statics(b, K=K, models=models, templates=orfs)
    return b, pl["os"], pl["os_null"], S0, models, orfs


def _rows(b, S0, o):
    """Rows in engine order (zero alignment slots), scaled so that the template's S/N is O(1)."""
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    rows = np.random.default_rng(2).standard_normal((6, b.ld))
    rows[:, ~live] = 0
    snr = OO.os_of_rows(b, S0, rows)["snr"][:, o]
    return rows / np.sqrt(np.sqrt(np.mean(snr**2)))


CASES = [(src, tm) for src in ("small", "synthetic") for tm in (False, True)]


@pytest.mark.parametrize("src,tm", CASES)
@pytest.mark.parametrize("method", ["phase_shift", "sky_scramble"])
def test_plan_statics_match_dense_oracle(src, tm, method):
    b, po, pn, S0, models, orfs = _setup(src, tm, method)
    o = pn["template"]
    rows = _rows(b, S0, o)
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ S0["C"][i] for i in range(b.n_psr)], axis=1)
    U = u_of_x(X * np.sqrt(S0["phi"]), po["pairs"], method)
    assert U.shape[1] == pn["kd"]
    got = U @ pn["V"][:NCOL + 1, :pn["kd"]].T / pn["dsqrt"]                   # [R, n + 1]
    ref = np.empty_like(got)
    ref[:, 0] = OO.os_of_rows(b, S0, rows)["snr"][:, o]
    for s in range(1, NCOL + 1):
        if method == "phase_shift":
            S = NO.phase_shifted_statics(b, pn["phases"][s - 1], K=K, models=models, templates=orfs)
            ref[:, s] = OO.os_of_rows(b, S, rows)["snr"][:, o]
        else:
            S = NO.scrambled_statics(S0, pn["radec"][s - 1], pn["template_name"])
            ref[:, s] = OO.os_of_rows(b, S, rows)["snr"][:, 0]
    d = float(np.max(np.abs(got - ref)))
    print(f"\n[os null] {method} {src} tm={tm}: max |dS/N| = {d:.1e} over {NCOL + 1} columns, max |S/N| "
          f"{np.max(np.abs(ref)):.1f}")
    assert d <= 1e-10
    assert np.all(pn["V"][:, pn["kd"]:] == 0) and np.all(pn["V"][NCOL + 1:] == 0)


@pytest.mark.parametrize("method,template", [("phase_shift", "hd"), ("phase_shift", "dipole"), ("phase_shift", 1),
                                             ("sky_scramble", "hd"), ("sky_scramble", "dipole")])
def test_column0_is_the_template(method, template):
    b = _batch(_synthetic(), tm=True)
    b.set_optimal_statistic(components=K)
    b.set_os_null(method, n=NCOL, seed=1, template=template)
    pl = b.plan()
    po, pn = pl["os"], pl["os_null"]
    o = po["names"].index(template) if isinstance(template, str) else template
    assert pn["template"] == o and pn["n_col"] == NCOL + 1 and pn["V"].shape[0] % 64 == 0 and pn["kdp"] % 32 == 0
    assert abs(pn["dsqrt"][0] / po["dsqrt"][o] - 1) <= 1e-14
    V0 = pn["V"][0, :pn["kd"]]
    if method == "phase_shift":
        assert np.array_equal(V0[0::2], np.repeat(po["orf"][o], K)) and np.all(V0[1::2] == 0)
        assert pn["phases"].shape == (NCOL, b.n_psr, K)
        assert np.all((pn["phases"] >= 0) & (pn["phases"] < 2 * np.pi))
    else:
        assert np.array_equal(V0, po["orf"][o])


@pytest.mark.parametrize("template", ["hd", "dipole"])
def test_scramble_matches_and_seeding(template):
    b = _batch(_synthetic())
    b.set_optimal_statistic(components=K)
    b.set_os_null("sky_scramble", n=16, seed=3, template=template, match=0.2)
    pn = b.plan()["os_null"]
    pa, pb = np.triu_indices(b.n_psr, 1)
    G = OO.hd_closed_form(b)[0 if template == "hd" else 1][pa, pb]
    for s in range(16):
        h, cz = NO.templates_at(pn["radec"][s])
        Gs = (h if template == "hd" else cz)[pa, pb]
        m = abs(G @ Gs) / np.sqrt((G @ G) * (Gs @ Gs))
        assert abs(m - pn["match"][s]) <= 1e-12 and m < 0.2
        assert np.allclose(pn["V"][1 + s, :len(pa)], Gs, rtol=0, atol=1e-13)
    ra, dec = pn["radec"][..., 0], pn["radec"][..., 1]
    assert np.all((ra >= 0) & (ra < 2 * np.pi)) and np.all(np.abs(dec) <= np.pi / 2)
    again = b.plan()["os_null"]
    assert np.array_equal(again["radec"], pn["radec"]) and np.array_equal(again["V"], pn["V"])
    b.set_os_null("sky_scramble", n=16, seed=4, template=template, match=0.2)
    assert not np.array_equal(b.plan()["os_null"]["radec"], pn["radec"])
    b.set_os_null("sky_scramble", n=16, seed=3, template=template, match=None)
    free = b.plan()["os_null"]
    assert free["attempts"] == 16
    # phase shifts: same seed, same set; another seed, another set
    b.set_os_null("phase_shift", n=4, seed=3, template=template)
    p1 = b.plan()["os_null"]["phases"]
    assert np.array_equal(p1, b.plan()["os_null"]["phases"])
    b.set_os_null("phase_shift", n=4, seed=4, template=template)
    assert not np.array_equal(p1, b.plan()["os_null"]["phases"])


def test_registration_lifecycle():
    b = _batch(_synthetic())
    b.set_optimal_statistic(components=K)
    b.set_os_null("phase_shift", n=4)
    assert b.plan()["os_null"] is not None and b.os_null_setup_s >= 0
    d0 = b.plan()["os_null"]["dsqrt"].copy()
    b._compiled = object()
    b.set_red(1, -12.5, 4.0, components=20)                     # a recipe change re-derives the null statics
    assert b._compiled is None
    assert not np.allclose(d0, b.plan()["os_null"]["dsqrt"])
    b._compiled = object()
    b.set_os_null("sky_scramble", n=4)
    assert b._compiled is None
    b.set_optimal_statistic(components=K)                       # clears the null registration
    assert b.plan()["os_null"] is None


def test_value_errors():
    b = _batch(_synthetic())
    with pytest.raises(ValueError, match="set_optimal_statistic"):
        b.set_os_null()
    b.set_optimal_statistic(components=K, orfs=("hd", "monopole", "dipole", np.eye(4) + 0.25))
    with pytest.raises(ValueError, match="unknown null method"):
        b.set_os_null("bootstrap")
    for bad in (0, -1, 65537, 2.5, True):
        with pytest.raises(ValueError, match="n must be"):
            b.set_os_null(n=bad)
    b.set_os_null(n=65536)                                       # the stated limit itself is accepted
    for bad in ("quadrupole", 4, -1, 1.0, None):
        with pytest.raises(ValueError, match="not registered"):
            b.set_os_null(template=bad)
    for bad in ("monopole", 1, "matrix", 3):
        with pytest.raises(ValueError, match="unchanged or undefined"):
            b.set_os_null("sky_scramble", template=bad)
    b.set_os_null("phase_shift", template="matrix")               # a phase shift of any template is defined
    for bad in (0.0, -0.1, 1.5, np.nan):
        with pytest.raises(ValueError, match="match"):
            b.set_os_null("sky_scramble", match=bad)
    b.set_os_null("sky_scramble", match=1.0)
    b.set_os_null("sky_scramble", match=None)
    # no n acceptances within 1000 n attempts
    t = _batch(_synthetic())
    t.set_optimal_statistic(components=K)
    t.set_os_null("sky_scramble", n=2, match=1e-9)
    with pytest.raises(ValueError, match="attempts"):
        t.plan()
