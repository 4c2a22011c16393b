"""GPU tests of the batched engine (PulsarBatch): epoch-compressed evaluation against the oracle with
injected draws, the throughput (Philox) mode against the oracle fed with the numpy restatement of the
same stream, shard / chunk invariance, and distributional properties at benchmark size."""
import numpy as np
import pytest

from oracle import philox as PH
from oracle import refnumpy as O
from tests.fixtures import load_flags_case, rel_rms

pytestmark = pytest.mark.gpu

TRIG = 1e-11          # see tests/test_gpu_parity.py
PHILOX = 2e-5         # fp32 MUFU Box-Muller on the GPU vs float64 log/sin/cos of the same fp32 uniforms in the oracle


def _batch(api_psrs, spec, **kw):
    from pta_replicator_b200.engine import PulsarBatch
    b = PulsarBatch(api_psrs, **kw)
    for i, s in enumerate(spec):
        be = np.array(s["backends"])
        b.set_white(i, efac=s["efac"], log10_equad=s["l10_equad"], flagid="f", flags=be)
        b.set_ecorr(i, s["l10_ecorr"], flagid="f", flags=be, coarsegrain=1.0 / 86400.0)
        b.set_red(i, s["rn_l10A"], s["rn_gamma"], components=30)
    b.set_gwb(-14.2, 13.0 / 3.0)
    b.add_cgw(gwtheta=1.1, gwphi=4.0, mc=3e9, dist=40.0, fgw=2.2e-8, phase0=1.3, psi=0.4, inc=1.0, pdist=1.3,
              tref=53000 * 86400)
    return b


def _psrs(spec):
    import pta_replicator_b200 as P
    out = []
    for s in spec:
        p = P.pulsar_from_arrays(s["name"], s["loc"], s["mjd"].astype(np.longdouble), s["err_us"],
                                 flags=[{"f": f, "pta": "SYN"} for f in s["flag"]])
        P.make_ideal(p)
        out.append(p)
    return out


def _oracle_total(b, spec, r, z1, z2, zb, zrn, gwb_per_psr, cgw):
    """Reference sum for realization r; draws are in ENGINE order (z1, z2) / bucket order (zb)."""
    st = b.compile()
    boff = st["psr_bucket_off"].cpu().numpy()
    out = []
    for i, s in enumerate(spec):
        n, off, o = b.ntoa[i], b.toa_off[i], b.order[i]
        zz1 = np.empty(n); zz1[o] = z1[r, off:off + n]
        zz2 = np.empty(n); zz2[o] = z2[r, off:off + n]
        ef = O.per_toa_params(s["efac"], s["backends"], s["flag"], n)
        eq = O.per_toa_params(10 ** s["l10_equad"], s["backends"], s["flag"], n)
        tot = O.white_noise(s["err_us"] * 1e-6, ef, eq, zz1, zz2)
        bk, firsts = O.epoch_buckets(s["mjd"], 1.0 / 86400.0)
        ec = O.ecorr_per_bucket(10 ** s["l10_ecorr"], s["backends"], s["flag"], firsts)
        tot = tot + O.jitter(bk, ec, zb[r, boff[i]:boff[i] + len(firsts)])
        tot = tot + O.red_noise(s["mjd"], s["rn_l10A"], s["rn_gamma"], zrn[r, i])
        tot = tot + gwb_per_psr[i] + cgw[i]
        out.append(tot)
    return out


def _cgw_oracle(spec):
    return [O.cgw(s["mjd"], s["loc"], 1.1, 4.0, 3e9, 40.0, 2.2e-8, 1.3, 0.4, 1.0, pdist=1.3, tref=53000 * 86400) for s in spec]


@pytest.mark.parametrize("exact", [False, True])
def test_injected_draws_all_signals_epoch_mode(exact):
    """All five terms at once, R = 6, draws injected.  exact=False exercises the in-epoch Taylor step
    (sub-banded epochs, nd = 3); exact=True evaluates every TOA as its own epoch."""
    import torch
    _, spec = load_flags_case()
    psrs = _psrs(spec)
    b = _batch(psrs, spec, exact_epochs=exact, rn_taylor_tol=1e-14)       # 1e-14 forces the 3-term Taylor step (nd = 3)
    st = b.compile()
    if not exact:
        assert st["n_epochs"] < 0.3 * b.n_toa_total and int(st["tiles_host"][:, 6].max()) == 3
        assert int(_batch(psrs, spec).compile()["tiles_host"][:, 6].max()) == 2    # the default tolerance (1e-13): 2 terms
    R, P = 6, len(spec)
    rng = np.random.default_rng(5)
    Jg = st["gwb_T_Jreal"]
    z1 = rng.standard_normal((R, b.ld)); z2 = rng.standard_normal((R, b.ld))
    zb = rng.standard_normal((R, st["n_bucket_total"])); zrn = rng.standard_normal((R, P, 60))
    zg = rng.standard_normal((R, P, Jg))
    out = b.generate(R, inject=dict(z1=torch.from_numpy(z1), z2=torch.from_numpy(z2), zb=torch.from_numpy(zb),
                                    zrn=torch.from_numpy(zrn), gwb_z=torch.from_numpy(zg))).cpu().numpy()
    g = b._gwb
    Nf = g["Nf"]
    M = np.linalg.cholesky(g["ORF"])
    cgw = _cgw_oracle(spec)
    worst = 0.0
    for r in range(R):
        w = np.zeros((P, Nf), complex)
        w[:, 1:Nf - 1] = zg[r, :, 0::2] + 1j * zg[r, :, 1::2]
        gw, _ = O.gwb_from_draws(dict(npts=g["npts"], dt=g["dt"], ut=g["ut"]), g["C"], M, w, [s["mjd"] for s in spec])
        ref = _oracle_total(b, spec, r, z1, z2, zb, zrn, gw, cgw)
        for i in range(P):
            worst = max(worst, rel_rms(b.unpack(out[r], i), ref[i]))
    assert worst < TRIG, worst


@pytest.mark.parametrize("merged", [False, True])
def test_throughput_mode_matches_oracle_fed_with_the_same_philox_stream(merged):
    """Philox mode end to end: the numpy restatement of the stream (oracle/philox.py) is pushed through
    the numpy oracle; the GWB uses the engine's own factor L (L L^T = T T^T is checked below).
    merged=True is the default throughput mode (one draw of variance w1^2 + w2^2 per TOA: the oracle's white term
    gets sqrt(efac^2 sigma^2 + (efac equad)^2) z1); merged=False draws z1 and z2 like the reference."""
    _, spec = load_flags_case()
    psrs = _psrs(spec)
    b = _batch(psrs, spec)
    b.white_merged = merged
    st = b.compile()
    R, P, seed, real0 = 8, len(spec), 987654321, 40
    out = b.generate(R, seed=seed, real0=real0).cpu().numpy()
    g = b._gwb
    L = st["gwb_L"].cpu().numpy()[:, :g["npts"]]
    M = np.linalg.cholesky(g["ORF"])
    boff = st["psr_bucket_off"].cpu().numpy()
    cgw = _cgw_oracle(spec)
    worst = 0.0
    for r in range(R):
        rid = real0 + r
        z1 = np.zeros((R, b.ld)); z2 = np.zeros((R, b.ld)); zb = np.zeros((R, st["n_bucket_total"])); zrn = np.zeros((R, P, 60))
        zg = np.zeros((P, g["npts"]))
        for i in range(P):
            n, off = b.ntoa[i], b.toa_off[i]
            z1[r, off:off + n] = PH.normals(PH.K_WHITE1, i, rid, n, seed)
            if merged:      # w1 z1 + w2 z2 with z2 := z1 * 0 and w1 := sqrt(w1^2 + w2^2): fold the ratio into z1
                pl = b.plan()
                w1p, w2p = pl["w1"][off:off + n], pl["w2"][off:off + n]
                z1[r, off:off + n] *= np.sqrt(w1p ** 2 + w2p ** 2) / w1p
            else:
                z2[r, off:off + n] = PH.normals(PH.K_WHITE2, i, rid, n, seed)
            nb = (boff[i + 1] if i + 1 < P else st["n_bucket_total"]) - boff[i]
            zb[r, boff[i]:boff[i] + nb] = PH.normals(PH.K_ECORR, i, rid, nb, seed)
            zrn[r, i] = PH.normals(PH.K_RED, i, rid, 60, seed)
            zg[i] = PH.normals(PH.K_GWB, i, rid, g["npts"], seed)
        grid = (M @ zg) @ L.T
        gw = [np.interp(s["mjd"] * 86400, g["ut"], grid[i]) for i, s in enumerate(spec)]
        ref = _oracle_total(b, spec, r, z1, z2, zb, zrn, gw, cgw)
        for i in range(P):
            worst = max(worst, rel_rms(b.unpack(out[r], i), ref[i]))
    assert worst < PHILOX, worst


def test_gwb_throughput_factor_has_the_reference_covariance():
    """L (npts x npts) used in throughput mode and T (npts x 2(Nf-2)), the reference's own linear map
    (pruned inverse DFT x sqrt(C)/dt), generate the same Gaussian law: L L^T == T T^T."""
    _, spec = load_flags_case()
    b = _batch(_psrs(spec), spec)
    st = b.compile()
    L = st["gwb_L"].cpu().numpy()
    T = st["gwb_T"].cpu().numpy()
    A, B = L @ L.T, T @ T.T
    assert np.linalg.norm(A - B) / np.linalg.norm(B) < 1e-12
    assert np.allclose(np.triu(L[:, :L.shape[0]], 1), 0.0)


def test_shards_and_chunks_are_bitwise_reproducible():
    """A realization depends only on (seed, global id): any split over calls / chunks / GPUs is identical."""
    import torch
    _, spec = load_flags_case()
    b = _batch(_psrs(spec), spec)
    full = b.generate(40, seed=3, real0=8)
    a = b.generate(16, seed=3, real0=8)
    c = b.generate(24, seed=3, real0=24)
    assert torch.equal(full[:16], a) and torch.equal(full[16:], c)
    b.default_chunk = 12
    d = b.generate(40, seed=3, real0=8)
    assert torch.equal(full, d)
    e = b.generate(40, seed=4, real0=8)
    assert not torch.equal(full, e)
    b.split_epoch = True                      # epoch kernel + TOA kernel: same arithmetic, same bits
    b.default_chunk = 512
    b._job_cache_key = None
    assert torch.equal(b.generate(40, seed=3, real0=8), full)
    b.split_epoch = False
    b._job_cache_key = None
    wide = b.generate(40, seed=3, real0=8, rc=32)          # 512-thread CTAs, 32 realizations each
    assert torch.equal(full, wide)
    h = b.generate_to_host(40, seed=3, real0=8, chunk=16)
    assert torch.equal(full.cpu(), h)


@pytest.mark.parametrize("exact", [False, True])
def test_two_kernel_schedule_is_bitwise_the_fused_generator(exact):
    """epoch kernel (tile x 32 realizations, ptar.cu launch_epoch) + TOA kernel against the fused kernel: same
    summation order, so every realization count (odd numbers of 16-realization blocks, partial blocks), the
    Philox mode and the injected mode must agree bit for bit; signal subsets exercise the flag paths."""
    import torch
    from pta_replicator_b200.engine import PulsarBatch
    _, spec = load_flags_case()
    psrs = _psrs(spec)

    def both(b, n, **kw):
        b.split_epoch = False
        b._job_cache_key = None
        x = b.generate(n, **kw)
        b.split_epoch = True
        b._job_cache_key = None
        y = b.generate(n, **kw)
        b.split_epoch = False
        b._job_cache_key = None
        return x, y

    b = _batch(psrs, spec, exact_epochs=exact)
    for n in (1, 5, 16, 17, 33, 48, 70):
        x, y = both(b, n, seed=11, real0=4)
        assert torch.equal(x, y), n
    st = b.compile()
    R, P = 19, len(spec)
    rng = np.random.default_rng(6)
    inj = dict(z1=torch.from_numpy(rng.standard_normal((R, b.ld))), z2=torch.from_numpy(rng.standard_normal((R, b.ld))),
               zb=torch.from_numpy(rng.standard_normal((R, st["n_bucket_total"]))),
               zrn=torch.from_numpy(rng.standard_normal((R, P, 60))),
               gwb_z=torch.from_numpy(rng.standard_normal((R, P, st["gwb_T_Jreal"]))))
    x, y = both(b, R, inject=inj)
    assert torch.equal(x, y)
    # subsets: ECORR only (no GEMM), red noise only, GWB only
    for which in ("ecorr", "red", "gwb"):
        s = PulsarBatch(psrs, exact_epochs=exact)
        for i in range(P):
            if which == "ecorr":
                s.set_ecorr(i, log10_ecorr=-6.3)
            elif which == "red":
                s.set_red(i, -13.5, 3.3, components=30)
        if which == "gwb":
            s.set_gwb(-14.0, 4.0)
        x, y = both(s, 21, seed=2)
        assert torch.equal(x, y) and float(x.abs().max()) > 0, which


def test_two_kernel_schedule_with_32_realization_blocks_and_scratch_checks():
    """rc = 32 in the two-kernel schedule writes 98-double rows (gen_css(32)), not 50: the engine sizes Cbuf from the
    effective rc, the library refuses a scratch that is too small, and the result equals the fused kernel's bit for bit
    on realization counts that leave ragged 32-blocks (ADVICE round 1: out-of-bounds Cbuf at n = 40, 16, 48, 80)."""
    import ctypes as C
    import torch
    from pta_replicator_b200 import _cabi
    _, spec = load_flags_case()
    b = _batch(_psrs(spec), spec)
    for n in (16, 40, 48, 80, 33):
        ref = b.generate(n, seed=9, real0=4)
        b.split_epoch = True
        got = b.generate(n, seed=9, real0=4, rc=32)
        b.split_epoch = False
        assert torch.equal(ref, got), n
    # a scratch sized for rc = 16 is rejected for rc = 32 instead of being overrun
    b.split_epoch = True
    st = b.compile()
    job, keep = b._job(st, 40, 9, None, 32)
    g = job.gen
    g.cbuf_len = int(st["tiles_host"][:, 4].sum()) * 3 * 50
    g.real0, g.nreal = 4, 40
    out = torch.empty((40, b.ld), dtype=torch.float64, device=b.device)
    g.out = out.data_ptr()
    if st["flags"] & _cabi.F_GWB:
        g.G = job.Gbuf
    rc = _cabi.lib().ptar_generate(C.byref(g), _cabi.current_stream())
    assert rc == -2 and b"Cbuf too small" in _cabi.lib().ptar_last_error()
    b.split_epoch = False


def test_cached_two_kernel_job_owns_its_epoch_scratch():
    """generate -> generate_to_host -> generate in the two-kernel schedule: the job generate caches owns its Cbuf (the
    epoch kernel's scratch is in that job's keep list), so the job generate_to_host builds in between cannot release it,
    and both generate calls give the fused schedule's bits."""
    import torch
    _, spec = load_flags_case()
    b = _batch(_psrs(spec), spec)
    fused = b.generate(40, seed=3, real0=8)
    b.split_epoch = True
    first = b.generate(40, seed=3, real0=8)
    host = b.generate_to_host(40, seed=3, real0=8, chunk=16)
    second = b.generate(40, seed=3, real0=8)
    assert torch.equal(first, fused) and torch.equal(second, fused) and torch.equal(host, fused.cpu())
    job, keep, _ = b._job_cache
    assert job.gen.Cbuf and job.gen.Cbuf in [t.data_ptr() for t in keep]


def test_parity_mode_requires_draws_for_every_enabled_term():
    """inject= with a term missing must raise instead of silently drawing that term from Philox (ADVICE round 1)."""
    import torch
    _, spec = load_flags_case()
    b = _batch(_psrs(spec), spec)
    st = b.compile()
    R, P = 2, len(spec)
    zg = torch.zeros((R, P, st["gwb_T_Jreal"]), dtype=torch.float64)
    with pytest.raises(ValueError, match="missing: z1, z2, zb, zrn"):
        b.generate(R, inject=dict(gwb_z=zg))


def test_gwb_factor_with_fewer_frequencies_than_grid_points():
    """howml = 1 gives 2 (Nf - 2) < npts: the throughput factor L is lower trapezoidal with that many columns
    (ADVICE round 1: shape error) and still has the reference covariance T T^T."""
    from pta_replicator_b200.engine import PulsarBatch
    _, spec = load_flags_case()
    b = PulsarBatch(_psrs(spec))
    b.set_gwb(-14.0, 13.0 / 3.0, howml=1)
    st = b.compile()
    assert st["gwb_T_Jreal"] < st["npts"]
    L, T = st["gwb_L"].cpu().numpy(), st["gwb_T"].cpu().numpy()
    A, B = L @ L.T, T @ T.T
    assert np.linalg.norm(A - B) / np.linalg.norm(B) < 1e-12
    x = b.generate(8, seed=3)
    assert bool(np.isfinite(x.cpu().numpy()).all()) and float(x.abs().max()) > 0


def test_ragged_realization_counts():
    """nreal not a multiple of the Philox group (4), the CTA chunk (16) or the GWB chunk: a prefix of a
    longer run, bit for bit; single-pulsar / single-signal batches; a chunk that is not a multiple of 16."""
    import torch
    from pta_replicator_b200.engine import PulsarBatch
    _, spec = load_flags_case()
    psrs = _psrs(spec)
    b = _batch(psrs, spec)
    full = b.generate(64, seed=21, real0=4)
    for n in (1, 3, 5, 17, 37, 63):
        assert torch.equal(b.generate(n, seed=21, real0=4), full[:n]), n
    b.default_chunk = 20                      # chunks of 20 realizations: 16 + 4 per CTA column
    assert torch.equal(b.generate(64, seed=21, real0=4), full)
    host = b.generate_to_host(37, seed=21, real0=4, chunk=12)
    assert torch.equal(host, full[:37].cpu())
    one = PulsarBatch(psrs[:1])
    one.set_gwb(-14.0, 4.0)
    x = one.generate(7, seed=1)
    assert torch.isfinite(x).all() and x.shape == (7, one.ld) and float(x.abs().max()) > 0
    with pytest.raises(Exception, match="multiple of 4"):
        b.generate(8, seed=21, real0=2)


def test_distribution_white_ecorr_and_merged_draw():
    """Per-TOA variance of white + ECORR over 4096 realizations; the single-draw variant (PTAR_F_WHITE1)
    has the same variance; an ECORR-only run is constant inside an epoch with variance ecorr^2."""
    from pta_replicator_b200.engine import PulsarBatch
    _, spec = load_flags_case()
    psrs = _psrs(spec)
    R = 4096

    def epoch_of_toa(b, pl):
        e = np.zeros(b.ld, dtype=np.int64)
        for t in pl["tiles"]:
            e[t[0]:t[0] + t[1]] = t[3] + pl["eloc"][t[0]:t[0] + t[1]]
        return e

    stats = []
    for merged in (False, True):
        b = PulsarBatch(psrs)
        b.white_merged = merged
        for i, s in enumerate(spec):
            be = np.array(s["backends"])
            b.set_white(i, efac=s["efac"], log10_equad=s["l10_equad"], flagid="f", flags=be)
            b.set_ecorr(i, s["l10_ecorr"], flagid="f", flags=be, coarsegrain=1.0 / 86400.0)
        x = b.generate(R, seed=11 + merged)
        pl = b.plan()
        var_expect = pl["w1"] ** 2 + pl["w2"] ** 2 + pl["ep_ecorr"][epoch_of_toa(b, pl)] ** 2
        real = pl["w1"] > 0
        v = x.var(dim=0, unbiased=True).cpu().numpy()
        ratio = v[real] / var_expect[real]
        assert abs(ratio.mean() - 1) < 3e-3 and ratio.std() < 3.5 * np.sqrt(2.0 / R)
        assert abs(x.mean().item()) < 1e-7
        stats.append(ratio.mean())
    assert abs(stats[0] - stats[1]) < 5e-3
    b = PulsarBatch(psrs)
    for i, s in enumerate(spec):
        b.set_ecorr(i, s["l10_ecorr"], flagid="f", flags=np.array(s["backends"]), coarsegrain=1.0 / 86400.0)
    x = b.generate(R, seed=13).cpu().numpy()
    pl = b.plan()
    e = epoch_of_toa(b, pl)
    for i in range(b.n_psr):
        sl = slice(b.toa_off[i], b.toa_off[i] + b.ntoa[i])
        ee, xx = e[sl], x[:, sl]
        same = ee[1:] == ee[:-1]
        assert np.array_equal(xx[:, 1:][:, same], xx[:, :-1][:, same])       # one draw per epoch
        ratio = xx.var(axis=0, ddof=1) / pl["ep_ecorr"][ee] ** 2
        assert abs(ratio.mean() - 1) < 0.02


def test_hd_correlation_of_the_gwb():
    """Cross-pulsar correlation of the throughput-mode GWB equals ORF_ab / sqrt(ORF_aa ORF_bb)."""
    from pta_replicator_b200.engine import PulsarBatch
    _, spec = load_flags_case()
    psrs = _psrs(spec)
    b = PulsarBatch(psrs)
    b.set_gwb(-14.0, 13.0 / 3.0)
    R = 8192
    x = b.generate(R, seed=5)
    orf = b._gwb["ORF"]
    # compare at (nearly) common epochs: use the grid directly through one TOA per pulsar near mid-span
    idx = []
    for i in range(len(psrs)):
        t = b.mjd[i]
        idx.append(b.toa_off[i] + int(np.argmin(np.abs(t - 55900.0))))
    y = x[:, idx].cpu().numpy()
    c = np.corrcoef(y.T)
    for a in range(len(psrs)):
        for bb in range(a + 1, len(psrs)):
            expect = orf[a, bb] / np.sqrt(orf[a, a] * orf[bb, bb])
            assert abs(c[a, bb] - expect) < 0.06, (a, bb, c[a, bb], expect)
