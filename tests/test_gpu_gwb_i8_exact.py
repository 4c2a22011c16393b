"""GPU test of the int8 GWB synthesis (ptar_gwb_synth_i8) for bit identity: the grid G is rebuilt on the host from the
device's own digit bytes (ZS, AS) and scales and must equal the device's G exactly.

The host reference is what the kernel computes by construction: per tile and diagonal d the exact integer sum over the
slice pairs s + t = d (every partial sum is an integer below 2^53, so a float64 matmul is exact in any order), then the
fp64 fold v = v + D_d 2^(-8 d) for d = 0 .. 6 in that order (D_d 2^(-8 d) is exact, so each step rounds like the device's
fma), then the product with the column scale sA * 2^-16 * sZ.  Any tile shape, k-chunk count or split of the slice
pairs between warpgroups must leave every bit of G unchanged."""
import numpy as np
import pytest

from tests import generator_reference as GR

pytestmark = pytest.mark.gpu

GWB = dict(log10_amplitude=-14.5, spectral_index=13.0 / 3.0, npts=150, howml=3)          # J = 152: J % 32 != 0
GWB_SMALL = dict(log10_amplitude=-14.5, spectral_index=13.0 / 3.0, npts=20, howml=1)     # J < 32, trapezoidal L


def _device_grid(b, R, seed=5, real0=8):
    """Digits of the Philox mix (fused for <= 72 pulsars, else mix + slicing), then G by ptar_gwb_synth_i8."""
    import torch
    from pta_replicator_b200 import _cabi
    L, s = _cabi.lib(), _cabi.current_stream()
    st = b.compile()
    job, keep = b._job(st, (R + 3) // 4 * 4, seed, None, 0)
    P = b.n_psr
    if P <= _cabi.MIX_I8_MAX_PSR:
        _cabi.check(L.ptar_gwb_mix_i8(job.ZS, job.M, job.zinv, P, job.Jg, job.Jpad, R, job.rcap, seed, real0, s), "mix_i8")
    else:
        _cabi.check(L.ptar_gwb_mix(job.Zm, job.M, None, P, job.Jg, R, seed, real0, s), "mix")
        _cabi.check(L.ptar_gwb_slice_i8(job.ZS, job.Zm, job.zinv, P, job.Jg, job.Jpad, R, job.rcap, s), "slice")
    ldr = job.gen.g_ldr
    G = torch.full((st["g_ld"] * ldr,), float("nan"), dtype=torch.float64, device=b.device)
    _cabi.check(L.ptar_gwb_synth_i8(G.data_ptr(), st["g_ld"], ldr, job.AS, job.colscale, job.ZS, job.zscale, P, job.Jg,
                                    job.Jpad, R, job.rcap, job.tile_list_i8, job.n_syn_tiles_i8, s), "synth_i8")
    torch.cuda.synchronize()
    ZS = next(k for k in keep if k.data_ptr() == job.ZS)
    return G.view(-1, ldr)[:, :R].cpu(), ZS.cpu().numpy(), job, st


def _host_grid(ZS, st, job, P, R):
    """G [g_ld, R] from the digit bytes, exactly as the kernel combines them."""
    import torch
    from pta_replicator_b200 import _cabi
    NS, BK = _cabi.I8_SLICES, _cabi.I8_BK
    Jpad, rcap, J = job.Jpad, job.rcap, job.Jg
    nk = Jpad // BK
    AS = st["i8_AS"].cpu().numpy()
    tiles = st["i8_tiles"].cpu().numpy()
    BN = AS.size // (len(tiles) * nk * NS * BK)
    A = AS.reshape(len(tiles), nk, NS, BN // 8, 2, 8, 16).transpose(0, 2, 3, 5, 1, 4, 6).reshape(len(tiles), NS, BN, Jpad)
    Z = ZS[:NS * P * rcap * Jpad].reshape(NS, P, rcap // 128, nk, 16, 2, 8, 16).transpose(0, 1, 2, 4, 6, 3, 5, 7)
    Z = Z.reshape(NS, P, rcap, Jpad)
    colscale, zscale = st["i8_colscale"].cpu().numpy(), st["i8_zscale"].cpu().numpy()
    G = np.full((st["g_ld"], R), np.nan)
    for p in range(P):
        idx = np.flatnonzero(tiles[:, 0] == p)
        if len(idx) == 0:
            continue
        Ap = A[idx].astype(np.float64)                                      # [tile][t][n][j]
        # the kernel runs only the k-chunks up to the tile's k extent
        kch = (np.minimum(tiles[idx, 3], J) + BK - 1) // BK
        Ap *= (np.arange(Jpad)[None, :] < (kch * BK)[:, None])[:, None, None, :]
        Ap = Ap.transpose(1, 0, 2, 3).reshape(NS, len(idx) * BN, Jpad)
        Zp = Z[:, p, :R].astype(np.float64)
        v = np.zeros((R, len(idx) * BN))
        for d in range(7):
            D = sum(Zp[s] @ Ap[d - s].T for s in range(max(0, d - NS + 1), min(d, NS - 1) + 1))
            assert np.abs(D).max(initial=0.0) < 2.0 ** 31                    # the device's int32 accumulators
            v = v + D * 2.0 ** (-8 * d)
        for k, ti in enumerate(idx):
            _, kn0, cnt, _ = tiles[ti]
            kpad = (cnt + 1) & ~1
            scol = np.zeros(kpad)
            scol[:cnt] = colscale[kn0:kn0 + cnt] * zscale[p]
            G[kn0:kn0 + kpad] = (v[:, k * BN:k * BN + kpad] * scol[None, :]).T
    return torch.from_numpy(G)


def _check(b, R, tag, seed=5, real0=8):
    import torch
    G, ZS, job, st = _device_grid(b, R, seed, real0)
    ref = _host_grid(ZS, st, job, b.n_psr, R)
    assert not torch.isnan(ref).any(), f"{tag}: a grid column without a tile"
    bad = (G != ref).sum().item()
    assert torch.equal(G, ref), f"{tag}: {bad} of {G.numel()} grid values differ"


def test_partim_small_grid_is_bit_identical():
    import os
    from pta_replicator_b200 import load_from_directories, make_ideal
    from pta_replicator_b200.engine import PulsarBatch
    gold = os.path.join(os.path.dirname(__file__), "golden", "partim_small")
    psrs = load_from_directories(os.path.join(gold, "par"), os.path.join(gold, "tim"), num_psrs=3)
    for p in psrs:
        make_ideal(p)
    b = PulsarBatch(psrs)
    b.set_gwb(-14.0, 13.0 / 3.0)
    for R in (8, 65):
        _check(b, R, f"partim_small R={R}")


def test_ng15_full_grid_is_bit_identical():
    """The benchmark's batch at its 1000 realizations per step."""
    from pta_replicator_b200 import synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("full")
    b = PulsarBatch(psrs)
    synthetic.ng15_recipe(b, noise)
    _check(b, 1000, "ng15-full R=1000", seed=20250922, real0=0)


def _edge_batch(P, gwb):
    rng = np.random.default_rng(P)
    return GR.gen_batch(ntoas=tuple(int(n) for n in rng.integers(1, 30, P)), dense=(), white=False, ecorr=False, red=0,
                        gwb=gwb)


@pytest.mark.parametrize("P,gwb,R", [(1, "small", 1), (2, "full", 63), (73, "small", 65), (112, "full", 129),
                                     (3, "full", 1025), (9, "small", 64)])
def test_edge_shapes_grid_is_bit_identical(P, gwb, R):
    """P = 1 ... 112 (73+: mix + slicing), J < 32 and J % 32 != 0, tiles shorter than the tile width and odd column
    counts (few TOAs per pulsar), R around the 64-realization CTA and 128-row r-block edges."""
    b = _edge_batch(P, GWB_SMALL if gwb == "small" else GWB)
    _check(b, R, f"P={P} J={'<32' if gwb == 'small' else '152'} R={R}", seed=P, real0=4 * P)


def test_dense_edge_batch_grid_is_bit_identical():
    """The generator edge sweep's dense batch (1 ... 2101 TOAs per pulsar: full and partial tiles, knots at the first
    and last grid interval)."""
    b = GR.gen_batch(gwb=GWB)
    for R in (33, 129):
        _check(b, R, f"dense edge batch R={R}", seed=7, real0=4)
