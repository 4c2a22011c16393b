"""GPU edge sweep of the residual generator and the GWB stage -- ptar_gwb_mix[_i8], ptar_gwb_synth, ptar_gwb_synth_i8,
ptar_generate (fused, two-kernel, rc = 32; the six throughput builds and the injected build) -- against the
extended-precision reference of tests/generator_reference.py, every output within its rigorous componentwise bound.
Throughput (Philox) mode is checked on the device's own normal stream: ``ptar_philox_normals`` is first proven to give the
generator's draws bit for bit.  Also: the shared-memory limits of every schedule and of the mixing kernel are refused
on the host before anything launches, alignment slots are written as zeros, the ``ld`` tail of ``out`` is never
touched, poisoned padding of injected draws changes nothing, and pad grid columns are 0 in both syntheses."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from tests import generator_reference as GR

pytestmark = pytest.mark.gpu

REPORT = GR.Report()
GWB = dict(log10_amplitude=-14.5, spectral_index=13.0 / 3.0, npts=150, howml=3)
GWB_SMALL = dict(log10_amplitude=-14.5, spectral_index=13.0 / 3.0, npts=20, howml=1)      # J < 32, trapezoidal L


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[generator edges] per kernel family:\n  " + "\n  ".join(REPORT.lines()))


def _np(t):
    return t.detach().cpu().numpy()


def _philox(b, kind, psr, R, real0, n, seed):
    """[R, n] fp64 of the device's normals (kind, pulsar, realization real0 + r, index 0 .. n - 1)."""
    import torch
    from pta_replicator_b200 import _cabi
    out = torch.empty((R, max(n, 1)), dtype=torch.float32, device=b.device)
    L = _cabi.lib()
    for r in range(R):
        _cabi.check(L.ptar_philox_normals(out[r].data_ptr(), kind, psr, real0 + r, 0, n, seed, _cabi.current_stream()))
    return _np(out)[:, :n].astype(np.float64)


def _philox_draws(b, st, R, real0, seed, two):
    from pta_replicator_b200 import _cabi
    D = {}
    if st["flags"] & _cabi.F_WHITE:
        for key, kind in (("z1", _cabi.K_WHITE1),) + ((("z2", _cabi.K_WHITE2),) if two else ()):
            z = np.zeros((R, b.ld))
            for p in range(b.n_psr):
                z[:, b.toa_off[p]:b.toa_off[p] + b.ntoa[p]] = _philox(b, kind, p, R, real0, b.ntoa[p], seed)
            D[key] = z
    if st["flags"] & _cabi.F_ECORR:
        off = _np(st["psr_bucket_off"])
        ends = np.r_[off[1:], st["n_bucket_total"]]
        D["zb"] = np.concatenate([_philox(b, _cabi.K_ECORR, p, R, real0, int(ends[p] - off[p]), seed)
                                  for p in range(b.n_psr)], axis=1)
    if st["flags"] & _cabi.F_RED:
        D["zrn"] = np.stack([_philox(b, _cabi.K_RED, p, R, real0, st["J"], seed) for p in range(b.n_psr)], axis=1)
    if st["flags"] & _cabi.F_GWB:
        D["gwb"] = np.stack([_philox(b, _cabi.K_GWB, p, R, real0, st["gwb_L_J"], seed) for p in range(b.n_psr)], axis=1)
    return D


def _find(keep, ptr):
    return next(t for t in keep if t.data_ptr() == ptr)


def _run(b, R, seed=0, real0=0, inject=None, rc=0, out=None):
    """One chunk of generate, launch by launch (the unfused mix + slice route of the int8 synthesis): out [R, ld] and
    the device's Zm [P, R, Jg] and grid G [g_ld, R] (None without a GWB)."""
    import torch
    from pta_replicator_b200 import _cabi
    st = b.compile()
    L, s = _cabi.lib(), _cabi.current_stream()
    R4 = (R + 3) // 4 * 4
    job, keep = b._job(st, R4, seed, inject, rc)
    g = job.gen
    Zm = G = None
    if st["flags"] & _cabi.F_GWB:
        zin = job.gwb_zin if inject is not None else None
        _cabi.check(L.ptar_gwb_mix(job.Zm, job.M, zin, b.n_psr, job.Jg, R, g.seed, real0, s), "ptar_gwb_mix")
        if job.AS and inject is None:
            _cabi.check(L.ptar_gwb_slice_i8(job.ZS, job.Zm, job.zinv, b.n_psr, job.Jg, job.Jpad, R, job.rcap, s), "slice")
            _cabi.check(L.ptar_gwb_synth_i8(job.Gbuf, g.g_ld, g.g_ldr, job.AS, job.colscale, job.ZS, job.zscale, b.n_psr,
                                            job.Jg, job.Jpad, R, job.rcap, job.tile_list_i8, job.n_syn_tiles_i8, s), "i8")
        else:
            _cabi.check(L.ptar_gwb_synth(job.Gbuf, g.g_ld, g.g_ldr, job.A, job.lda, job.Zm, job.Jg, R, job.tile_list,
                                         job.n_syn_tiles, job.knots, job.lower_tri, s), "ptar_gwb_synth")
        g.G = job.Gbuf
        Zm = _np(_find(keep, job.Zm))[:b.n_psr * R * job.Jg].reshape(b.n_psr, R, job.Jg)
        G = _np(_find(keep, job.Gbuf)).reshape(st["g_ld"], -1)[:, :R]
    if out is None:
        out = torch.full((R, b.ld), float("nan"), dtype=torch.float64, device=b.device)
    g.real0, g.nreal, g.out = real0, R, out.data_ptr()
    _cabi.check(L.ptar_generate(C.byref(g), s), "ptar_generate")
    return out, Zm, G, job


def _statics(b, st, merged, G):
    from pta_replicator_b200 import _cabi
    S = {k: _np(st[k]) for k in ("w1", "w2", "wm", "dtau", "det", "ep_gidx", "ep_gw", "ep_ginv", "ep_ecorr", "ep_bucket",
                                 "psr_bucket_off")}
    S["eloc"] = _np(st["eloc"]).view(np.uint16)
    S.update(tiles=st["tiles_host"], J=st["J"], ld=b.ld, flags=st["flags"], G=G, conv=st.get("conv", 0))
    if merged and (st["flags"] & _cabi.F_WHITE):
        S["flags"] |= _cabi.F_WHITE1
        S["w1"] = S["wm"]
    if st["flags"] & _cabi.F_RED:
        S["Ftile"] = _np(st["Ftile"])
        S["rn_scale"] = _np(st["rn_scale"]).reshape(b.n_psr, st["J"])
        S["rn_omega"] = _np(st["rn_omega"]).reshape(b.n_psr, st["J"] // 2)
    return S


def _gwb_refs(b, st, R, Zm, G, z, inject, tag):
    """The mix against its reference on the draws ``z`` [R, P, Jg], the grid against the synthesis reference on the
    device's Zm; pad columns exactly 0."""
    from pta_replicator_b200 import _cabi
    Jg = Zm.shape[2]
    GR.check(Zm, GR.mix(_np(st["M"]), z[:, :, :Jg]), f"{tag} mix", REPORT, "mix")
    knots, tiles = _np(st["knots"]), _np(st["syn_tiles"])
    assert np.all(G[knots < 0] == 0.0), f"{tag}: pad grid columns"
    if inject is not None or not b.use_tcgen05:
        A = _np(st["gwb_T"] if inject is not None else st["gwb_L"]).reshape(-1, Jg)
        GR.check(G, GR.synth(A, Zm, knots, tiles), f"{tag} synth", REPORT, "synth_dmma")
    else:
        A = _np(st["gwb_L"]).reshape(-1, Jg)
        cs = _np(st["i8_colscale"])
        sA = np.ones(A.shape[0])
        sA[knots[knots >= 0]] = cs[knots >= 0] * 2.0 ** 16
        ref = GR.synth_i8(A, sA, Zm, _np(st["i8_zscale"]), knots, tiles)
        GR.check(G, ref, f"{tag} synth_i8", REPORT, "synth_i8")
        d = np.abs(G - ref["exact"])[knots >= 0]
        REPORT.add("i8_vs_exact", 0.0, float(d.max() / (GR.U * max(np.abs(ref["exact"]).max(), 1e-300))))


def _inject(b, st, R, seed, poison=False):
    """Injected draws; with ``poison`` the alignment slots and ld tail of z1 / z2 hold NaN, +inf, -inf."""
    import torch
    from pta_replicator_b200 import _cabi
    rng = np.random.default_rng(seed)
    D = dict(z1=rng.standard_normal((R, b.ld)), z2=rng.standard_normal((R, b.ld)),
             zb=rng.standard_normal((R, max(st["n_bucket_total"], 1))),
             zrn=rng.standard_normal((R, b.n_psr, max(st["J"], 2))))
    if st["flags"] & _cabi.F_GWB:
        D["gwb"] = np.zeros((R, b.n_psr, st["gwb_T_J"]))
        D["gwb"][:, :, :st["gwb_T_Jreal"]] = rng.standard_normal((R, b.n_psr, st["gwb_T_Jreal"]))
    if poison:
        pad = np.ones(b.ld, dtype=bool)
        for s, n in zip(b.toa_off, b.ntoa):
            pad[s:s + n] = False
        vals = np.array([np.nan, np.inf, -np.inf])[np.arange(pad.sum()) % 3]
        for k in ("z1", "z2"):
            D[k][:, pad] = vals[None, :]
    inj = {k: torch.from_numpy(D[k]) for k in ("z1", "z2", "zb", "zrn")}
    if st["flags"] & _cabi.F_GWB:
        inj["gwb_z"] = torch.from_numpy(D["gwb"][:, :, :st["gwb_T_Jreal"]])
    return D, inj


def _sweep(b, R, seed=0, real0=0, mode="philox", rc=0, tag=""):
    """generate (launch by launch) against the reference; the library's generate gives the same bits."""
    import torch
    from pta_replicator_b200 import _cabi
    st = b.compile()
    inject, D = None, None
    if mode == "inject":
        D, inject = _inject(b, st, R, seed)
    out, Zm, G, job = _run(b, R, seed, real0, inject, rc)
    got = _np(out)
    if mode == "philox":
        D = _philox_draws(b, st, R, real0, seed, two=not b.white_merged)
    if Zm is not None:
        _gwb_refs(b, st, R, Zm, G, D["gwb"], inject, tag)
    S = _statics(b, st, merged=(mode == "philox" and b.white_merged), G=G)
    ref, written = GR.generate(S, D, R)
    sched = "rc32" if rc == 32 else ("two_kernel" if b.split_epoch else "fused")
    GR.check(got[:, written], {k: v[:, written] for k, v in ref.items()}, f"{tag} generate", REPORT, f"gen_{sched}_{mode}")
    assert np.all(np.isnan(got[:, ~written])), f"{tag}: the ld tail was written"
    pad = written.copy()
    for s, n in zip(b.toa_off, b.ntoa):
        pad[s:s + n] = False
    assert np.all(got[:, pad] == 0.0), f"{tag}: alignment slots"
    lib_out = b.generate(R, seed=seed, real0=real0, inject=inject, chunk=R, rc=rc)
    assert torch.equal(lib_out[:, torch.from_numpy(written).to(lib_out.device)], out[:, torch.from_numpy(written).to(out.device)])
    return got, D


_BATCHES = {}


def _batch(key, **kw):
    if key not in _BATCHES:
        _BATCHES[key] = GR.gen_batch(**kw)
    b = _BATCHES[key]
    b.split_epoch, b.white_merged, b.use_tcgen05 = False, True, True
    return b


# (batch key, batch kwargs, R, real0, mode, schedule)
FULL = dict(gwb=GWB)
SWEEP = [
    ("full", FULL, 17, 0, "inject", "fused"),
    ("full", FULL, 33, 4, "philox", "fused"),
    ("full", FULL, 16, 2 ** 34 + 8, "philox", "two_kernel"),
    ("full", FULL, 129, 0, "philox", "rc32"),
    ("full", FULL, 3, 0, "inject", "two_kernel"),
    ("full", FULL, 33, 0, "inject", "rc32"),
    ("conv_tol14", dict(conv=True, red=31, gwb=GWB_SMALL, rn_taylor_tol=1e-14), 15, 4, "philox", "fused"),
    ("conv_tol14", dict(conv=True, red=31, gwb=GWB_SMALL, rn_taylor_tol=1e-14), 4, 0, "inject", "two_kernel"),
    ("exact_red1", dict(red=1, gwb=GWB_SMALL, exact_epochs=True), 127, 0, "philox", "two_kernel"),
    ("exact_red1", dict(red=1, gwb=GWB_SMALL, exact_epochs=True), 1, 0, "inject", "fused"),
    ("red2_det", dict(red=2, det=True, two_draws=True), 128, 8, "philox", "rc32"),
    ("red30_det", dict(red=30, det=True), 4, 0, "philox", "fused"),
]


@pytest.mark.parametrize("key,kw,R,real0,mode,sched", SWEEP)
def test_generator_edges(key, kw, R, real0, mode, sched):
    b = _batch(key, **kw)
    b.split_epoch = sched == "two_kernel"
    _sweep(b, R, seed=7, real0=real0, mode=mode, rc=32 if sched == "rc32" else 0, tag=f"{key} {mode} {sched} R={R}")


# the six throughput builds (WHITE 0 / 1 / 2 x DET 0 / 1) and the epoch-only subsets
BUILDS = [("w0d0", dict(white=False, red=3)), ("w0d1", dict(white=False, red=3, det=True)),
          ("w1d0", dict(red=3)), ("w1d1", dict(red=3, det=True)),
          ("w2d0", dict(red=3, two_draws=True)), ("w2d1", dict(red=3, two_draws=True, det=True)),
          ("ecorr_only", dict(white=False, red=0)), ("gwb_only", dict(white=False, ecorr=False, red=0, gwb=GWB_SMALL))]


@pytest.mark.parametrize("key,kw", BUILDS)
@pytest.mark.parametrize("sched", ["fused", "two_kernel", "rc32"])
def test_generator_builds(key, kw, sched):
    b = _batch("b_" + key, ntoas=(1, 5, 17, 1025), dense=(), **kw)
    b.white_merged = not kw.get("two_draws", False)
    b.split_epoch = sched == "two_kernel"
    _sweep(b, 17, seed=3, real0=4, mode="philox", rc=32 if sched == "rc32" else 0, tag=f"{key} {sched}")
    if sched == "fused":
        _sweep(b, 5, seed=3, mode="inject", tag=f"{key} inject")


def test_philox_normals_are_the_generators_draws():
    """White-only batch, no deterministic term: generate = w * n exactly (one merged draw) and fma(w2, n2, w1 n1) exactly
    (two draws), for both rc and both schedules' TOA stage -- so the sweep may use ptar_philox_normals as the draws."""
    b = _batch("white_only", ntoas=(1, 2, 3, 5, 17, 70), dense=(), ecorr=False, red=0, two_draws=True)
    st = b.compile()
    R, real0, seed = 9, 2 ** 34 + 8, 12345
    for merged in (True, False):
        b.white_merged = merged
        D = _philox_draws(b, st, R, real0, seed, two=not merged)
        w1, w2, wm = _np(st["w1"]), _np(st["w2"]), _np(st["wm"])
        if merged:
            want = wm[None, :] * D["z1"]
        else:
            p1 = w1[None, :] * D["z1"]
            want = np.array([[float(Fraction(a) + Fraction(c) * Fraction(d)) for a, c, d in zip(pr, w2, zr)]
                             for pr, zr in zip(p1, D["z2"])])
        for rc in (0, 32):
            got = _np(b.generate(R, seed=seed, real0=real0, rc=rc))
            mask = np.zeros(b.ld, dtype=bool)
            for s, n in zip(b.toa_off, b.ntoa):
                mask[s:s + n] = True
            assert np.array_equal(got[:, mask], want[:, mask]), (merged, rc)


@pytest.mark.parametrize("P", [1, 2, 3, 8, 9, 72, 73, 112])
@pytest.mark.parametrize("route", ["i8", "dmma", "parity"])
def test_gwb_stage_pulsar_counts(P, route):
    """Mix and synthesis at P = 1 ... 112 (73+: the unfused mix + slice route; 112: the largest the mix admits), both
    syntheses and the parity mode (gwb_T, lower_tri = 0); the generate output of a GWB-only batch within its bound."""
    rng = np.random.default_rng(P)
    ntoas = tuple(int(n) for n in rng.integers(1, 30, P))
    b = _batch(f"gwb_P{P}", ntoas=ntoas, dense=(), white=False, ecorr=False, red=0,
               gwb=GWB_SMALL if P % 2 else GWB)
    b.use_tcgen05 = route == "i8"
    R = 4 if P >= 72 else (1, 4, 17, 33, 128, 129)[P % 6]
    _sweep(b, R, seed=P, real0=4 * P, mode="inject" if route == "parity" else "philox", tag=f"P={P} {route}")


def test_large_R_and_mix_with_fewer_items_than_ctas():
    """R = 1025 (9 synthesis row blocks, a ragged last one) and R = 1 with one pulsar (one mix item for hundreds of
    resident CTAs)."""
    b = _batch("bigR", ntoas=(3, 64, 1025), dense=(), gwb=GWB)
    _sweep(b, 1025, seed=1, real0=0, mode="philox", tag="R=1025")
    b1 = _batch("gwb_P1", ntoas=(int(np.random.default_rng(1).integers(1, 30)),), dense=(), white=False, ecorr=False,
                red=0, gwb=GWB_SMALL)
    _sweep(b1, 1, seed=2, mode="philox", tag="P=1 R=1")


def test_poisoned_padding_and_preset_out():
    """NaN / +-inf in the alignment slots and the ld tail of injected z1 / z2 change no output; a preset out keeps its
    ld tail and gets zeros in the alignment slots."""
    import torch
    b = _batch("full", **FULL)
    st = b.compile()
    R = 6
    _, inj = _inject(b, st, R, seed=5)
    _, pinj = _inject(b, st, R, seed=5, poison=True)
    a = b.generate(R, inject=inj)
    c = b.generate(R, inject=pinj)
    assert torch.equal(a, c)
    out = torch.full((R, b.ld), 7.0, dtype=torch.float64, device=b.device)
    got = _np(_run(b, R, inject=inj, out=out)[0])
    used = b.toa_off[-1] + (b.ntoa[-1] + 3) // 4 * 4
    assert np.all(got[:, used:] == 7.0)
    assert np.array_equal(got[:, :used], _np(a)[:, :used])


def test_shared_memory_limits_are_refused_on_the_host():
    """J at each schedule's limit runs (258 fused rc = 16, 180 rc = 32, 154 two-kernel); J + 2 is refused by the engine
    (ValueError) and by the library (PtarError, before anything launches); a GWB over 112 pulsars is refused by compile()
    and by ptar_gwb_mix."""
    import torch
    from pta_replicator_b200 import _cabi
    assert (_cabi.max_red_columns(16), _cabi.max_red_columns(32), _cabi.max_red_columns(16, True)) == (258, 180, 154)
    for J, rc, split in ((258, 0, False), (180, 32, False), (154, 0, True), (180, 32, True)):
        b = GR.gen_batch(ntoas=(5, 40), dense=(), red=J // 2)
        b.split_epoch = split
        _sweep(b, 5, seed=J, mode="philox", rc=rc, tag=f"J={J} rc={rc} split={split}")
        st = b.compile()
        job, keep = b._job(st, 8, 0, None, rc)
        g = job.gen
        out = torch.empty((8, b.ld), dtype=torch.float64, device=b.device)
        g.nreal, g.out, g.J = 8, out.data_ptr(), J + 2
        assert _cabi.lib().ptar_generate(C.byref(g), _cabi.current_stream()) == -3
        assert b"too large for shared memory" in _cabi.lib().ptar_last_error()
    with pytest.raises(ValueError, match="does not fit shared memory"):
        b = GR.gen_batch(ntoas=(5, 40), dense=(), red=78)
        b.split_epoch = True
        b.generate(4)
    with pytest.raises(ValueError, match="limited to 129 components"):
        GR.gen_batch(ntoas=(5, 40), dense=(), red=130).compile()
    rng = np.random.default_rng(0)
    b = GR.gen_batch(ntoas=tuple(int(n) for n in rng.integers(1, 6, 113)), dense=(), white=False, ecorr=False, red=0,
                     gwb=GWB_SMALL)
    with pytest.raises(ValueError, match="limited to 112 pulsars"):
        b.compile()
    z = torch.empty(8 * 113 * 20, dtype=torch.float64, device=b.device)
    M = torch.zeros(113 * 113, dtype=torch.float64, device=b.device)
    assert _cabi.lib().ptar_gwb_mix(z.data_ptr(), M.data_ptr(), None, 113, 20, 8, 0, 0, _cabi.current_stream()) == -3
    assert b"more than 112 pulsars" in _cabi.lib().ptar_last_error()
