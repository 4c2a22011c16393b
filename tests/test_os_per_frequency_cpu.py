"""CPU tests of the per-frequency optimal statistic's host statics (``PulsarBatch.set_os_per_frequency``,
``plan()["os_pf"]``) against the dense oracle (tests/pfos_oracle.py), the statistic of some rows from the plan's
statics against the oracle's, the argument and frequency-naming checks, the registration's lifecycle and the ctypes
layout of ``ptar_os_pf_model``.  ``plan_only`` batches: the 3 ``partim_small`` pulsars and the synthetic multi-backend
case of test_optimal_statistic_cpu.py."""
import os
import re

import numpy as np
import pytest

from tests import os_oracle as OO
from tests import pfos_oracle as PO
from tests.test_optimal_statistic_cpu import _batch, _models, _small, _synthetic

# the optimal statistic's tolerance (test_optimal_statistic_cpu.py): Woodbury against dense null-space solves
TOL = 1e-10
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / np.max(np.abs(b)))


def _templates(src, n):
    if src == "small":
        return ("hd",) if n == 1 else ("hd", "monopole")
    if n == 1:
        return ("hd",)
    G = np.random.default_rng(4).uniform(-0.5, 0.5, (4, 4))
    return ("hd", "monopole", "dipole", G + G.T)


def _live(b):
    live = np.zeros(b.ld, dtype=bool)
    for i in range(b.n_psr):
        live[b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] = True
    return live


def _plan_of_rows(b, po, pp, rows):
    """The plan's statics applied in numpy to rows [R, ld]: what the kernel computes."""
    nc = po["nc"]
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :nc]
                  for i in range(b.n_psr)], axis=1)
    pa, pb = po["pairs"][:, 0], po["pairs"][:, 1]
    R, K = len(rows), pp["K"]
    d = (X[:, pa] * X[:, pb]).reshape(R, len(pa), K, 2).sum(axis=3).transpose(0, 2, 1)
    bo = np.einsum("oq,rkq->rok", po["orf"], d)
    return dict(rho=d / pp["t"], phi=bo / pp["dnorm"], snr=bo / pp["dsqrt"], phi_mc=np.einsum("kop,rpk->rok", pp["finv"], bo))


CASES = ([(src, tm, common, 10, 1) for src in ("small", "synthetic") for tm in (False, True) for common in (None, -14.5)]
         + [("small", True, None, 1, 2), ("synthetic", True, -14.5, 1, 4), ("small", False, None, 16, 2),
            ("synthetic", True, None, 16, 4), ("synthetic", False, -14.5, 10, 4)])


@pytest.mark.parametrize("src,tm,common,K,n_orf", CASES)
def test_statics_match_dense_oracle(src, tm, common, K, n_orf):
    b = _batch(_small() if src == "small" else _synthetic(), tm=tm)
    orfs = _templates(src, n_orf)
    b.set_optimal_statistic(components=K, orfs=orfs, log10_A_common=common)
    b.set_os_per_frequency()
    pl = b.plan()
    po, pp = pl["os"], pl["os_pf"]
    S = OO.statics(b, K=K, log10_A_common=common, models=_models(b) if tm else None, templates=orfs)
    T = PO.pf_statics(b, S)
    worst = dict(t=_rel(pp["t"], T["t"]), D=_rel(pp["dnorm"], T["D"]), Finv=max(_rel(pp["finv"][k], T["Finv"][k])
                                                                                 for k in range(K)))
    assert pp["K"] == K and pp["t"].shape == (K, len(S["pairs"][0])) and pp["finv"].shape == (K, len(orfs), len(orfs))
    assert np.array_equal(pp["freqs"], np.arange(1, K + 1) / b._os["Tspan"])
    assert _rel(pp["phi_tilde"], S["phi"][0::2]) <= 1e-14
    assert np.array_equal(pp["sigma"], 1 / np.sqrt(pp["t"])) and np.array_equal(pp["phi_sigma"], 1 / np.sqrt(pp["dnorm"]))
    # the outputs of some rows through the plan's statics against the oracle's
    rows = np.random.default_rng(1).standard_normal((3, b.ld)) * 1e-6
    rows[:, ~_live(b)] = 0
    got, ref = _plan_of_rows(b, po, pp, rows), PO.pf_of_rows(b, S, rows, T)
    worst["rho/sigma"] = float(np.max(np.abs(got["rho"] - ref["rho"]) * np.sqrt(T["t"])))
    worst["phi/sigma"] = float(np.max(np.abs(got["phi"] - ref["phi"]) * np.sqrt(T["D"])))
    worst["snr"] = float(np.max(np.abs(got["snr"] - ref["snr"])))
    sig_mc = np.sqrt(np.stack([np.diag(f) for f in T["Finv"]], axis=1))                     # [n_orf, K]
    worst["phi_mc/sigma"] = float(np.max(np.abs(got["phi_mc"] - ref["phi_mc"]) / sig_mc))
    print(f"\n[os pf statics] {src} tm={tm} common={common} K={K} n_orf={n_orf}: " +
          ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert max(worst.values()) < TOL, worst


def test_numerator_identity():
    """sum_k phi~_k b_ok, rebuilt from phi_ok D_ok, is the broadband numerator b_o = sum_q Gamma^o_q x_a . x_b."""
    b = _batch(_synthetic(), tm=True)
    b.set_optimal_statistic(components=12)
    b.set_os_per_frequency()
    pl = b.plan()
    po, pp = pl["os"], pl["os_pf"]
    rows = np.random.default_rng(3).standard_normal((4, b.ld)) * 1e-6
    rows[:, ~_live(b)] = 0
    got = _plan_of_rows(b, po, pp, rows)
    num = np.einsum("k,rok->ro", pp["phi_tilde"], got["phi"] * pp["dnorm"])
    mag = np.einsum("k,rok->ro", pp["phi_tilde"], np.abs(got["phi"] * pp["dnorm"]))
    X = np.stack([rows[:, b.toa_off[i]:b.toa_off[i] + b.ntoa[i]] @ po["C"][b.toa_off[i]:b.toa_off[i] + b.ntoa[i], :24]
                  for i in range(b.n_psr)], axis=1) * np.sqrt(po["phi"])
    d = np.einsum("rpj,rpj->rp", X[:, po["pairs"][:, 0]], X[:, po["pairs"][:, 1]])
    bo = d @ po["orf"].T
    assert np.max(np.abs(num - bo) / mag) < 1e-12


def _with_z(b, edit):
    """Make ``b.plan()`` see ``edit(Z)`` as the optimal statistic's Z (the per-frequency statics' only input from it)."""
    orig = b._plan_os

    def patched():
        po = orig()
        po["Z"] = edit(po["Z"].copy())
        return po
    b._plan_os = patched


def test_value_errors_name_the_frequency():
    b = _batch(_synthetic())
    with pytest.raises(ValueError, match="set_optimal_statistic"):
        b.set_os_per_frequency()
    b.set_optimal_statistic(components=6, orfs=("hd", "dipole"))
    b.set_os_per_frequency()
    # pulsar 2 has no power at f_3: every pair with it has t_q3 = 0

    def silence(Z):
        Z[2, 4:6, :] = 0.0
        return Z
    _with_z(b, silence)
    with pytest.raises(ValueError, match=r"pulsar pair \(0, 2\) .*frequency k = 3 \(f = "):
        b.plan()
    # at f_2 only the pair (0, 1) keeps its weight: F_2 of two templates has rank 1
    b2 = _batch(_synthetic())
    b2.set_optimal_statistic(components=6, orfs=("hd", "dipole"))
    b2.set_os_per_frequency()

    def starve(Z):
        Z[2:, 2:4, :] *= 1e-20
        return Z
    _with_z(b2, starve)
    with pytest.raises(ValueError, match=r"Fisher matrix F_k at k = 2 \(f = .*singular"):
        b2.plan()


def test_registration_lifecycle():
    b = _batch(_synthetic())
    b.set_optimal_statistic(components=8)
    b.set_os_anisotropy(lmax=1)
    b._compiled = object()
    b.set_os_per_frequency()
    assert b._compiled is None
    pl = b.plan()
    assert pl["os_pf"] is not None and b.os_pf_setup_s >= 0 and pl["os_pf"]["setup_s"] >= 0
    assert pl["os_aniso"] is not None
    t0 = pl["os_pf"]["t"].copy()
    b.set_red(1, -12.5, 4.0, components=20)            # a recipe change re-derives the statics
    assert not np.allclose(t0, b.plan()["os_pf"]["t"])
    b.set_optimal_statistic(components=8)              # clears the registration
    assert b.plan()["os_pf"] is None
    fresh = _batch(_synthetic())
    fresh.set_optimal_statistic(components=8)
    assert fresh.plan()["os_pf"] is None and fresh.os_pf_setup_s is None


def test_os_pf_model_layout_matches_the_header():
    import ctypes as C

    from pta_replicator_b200 import _cabi
    hdr = open(os.path.join(ROOT, "include", "ptar.h")).read()
    end = hdr.index("} ptar_os_pf_model;")
    body = hdr[hdr.rindex("typedef struct {", 0, end):end]
    fields = re.findall(r"^\s*((?:const )?[a-z0-9_]+\*?)\s+([a-z_0-9]+);", body, re.M)
    assert [n for _, n in fields] == [n for n, _ in _cabi.OsPfModel._fields_]
    for (ctype, name), (_, cls) in zip(fields, _cabi.OsPfModel._fields_):
        assert ctype == "const double*" and cls is C.c_void_p, name          # four device pointers
    assert C.sizeof(_cabi.OsPfModel) == 8 * len(fields)
    assert [getattr(_cabi.OsPfModel, n).offset for _, n in fields] == [8 * i for i in range(len(fields))]
