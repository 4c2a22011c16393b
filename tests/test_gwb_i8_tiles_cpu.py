"""CPU tests of the tile list of the int8 GWB synthesis (``PulsarBatch.i8_tiles``): on plan_only batches every compact grid
column is computed by exactly one tile, a tile holds one pulsar's consecutive columns, at most I8_BN of them, and its k
extent reaches past its last knot (L is lower triangular, so the k-chunks beyond it multiply zeros)."""
import numpy as np
import pytest

from tests import generator_reference as GR

GWB = dict(log10_amplitude=-14.5, spectral_index=13.0 / 3.0, npts=150, howml=3)
GWB_SMALL = dict(log10_amplitude=-14.5, spectral_index=13.0 / 3.0, npts=20, howml=1)


def _check_tiles(pl, tiles, bn):
    knots, syn = pl["knots"], pl["syn_tiles"]
    g_ld = pl["g_ld"]
    assert tiles.dtype == np.int32 and tiles.shape[1] == 4
    written = np.zeros(g_ld, dtype=np.int64)
    for p, kn0, cnt, kend in tiles.tolist():
        assert 1 <= cnt <= bn
        kpad = (cnt + 1) & ~1                     # the kernel also writes the pad column of an odd count (as a zero)
        written[kn0:kn0 + kpad] += 1
        mine = syn[syn[:, 0] == p]
        assert mine[:, 1].min() <= kn0 and kn0 + cnt <= (mine[:, 1] + mine[:, 2]).max(), "a tile crosses pulsars"
        assert kend == knots[kn0 + cnt - 1] + 1 and np.all(knots[kn0:kn0 + cnt] < kend)
    assert np.all(written == 1), "every compact column exactly once"
    # pulsar-major, ascending columns; one short tile per pulsar at most
    assert np.all(np.diff(tiles[:, 1]) > 0) and np.all(np.diff(tiles[:, 0]) >= 0)
    for p in np.unique(tiles[:, 0]):
        assert np.sum(tiles[tiles[:, 0] == p, 2] < bn) <= 1


@pytest.mark.parametrize("bn", [32, 48])
@pytest.mark.parametrize("kw", [dict(gwb=GWB), dict(gwb=GWB_SMALL, red=3), dict(ntoas=(1, 2, 3, 5, 17, 70), dense=(), gwb=GWB)],
                         ids=["edges", "J<32", "short"])
def test_int8_tiles_cover_every_knot_once(kw, bn):
    from pta_replicator_b200.engine import PulsarBatch
    b = GR.gen_batch(plan_only=True, **kw)
    pl = b.plan()
    tiles = PulsarBatch.i8_tiles(pl["knots"], pl["syn_tiles"], bn)
    _check_tiles(pl, tiles, bn)
    assert np.any(tiles[:, 2] < bn)                                  # tiles shorter than bn occur


def test_int8_tiles_of_ng15_full():
    """The benchmark's batch: 48-knot tiles cut from each pulsar's whole column range need fewer k-chunks than 48-knot
    tiles cut from the 64-column synthesis tiles would."""
    from pta_replicator_b200 import _cabi, synthetic
    from pta_replicator_b200.engine import PulsarBatch
    psrs, noise = synthetic.make_ng15_like("full")
    b = PulsarBatch(psrs, plan_only=True)
    synthetic.ng15_recipe(b, noise)
    pl = b.plan()
    tiles = PulsarBatch.i8_tiles(pl["knots"], pl["syn_tiles"])
    _check_tiles(pl, tiles, _cabi.I8_BN)
    J = b._gwb["npts"]
    chunks = lambda kend: (np.minimum(kend, J) + _cabi.I8_BK - 1) // _cabi.I8_BK
    per_64 = [(kn0 + n0, min(_cabi.I8_BN, cnt - n0)) for _, kn0, cnt, _ in pl["syn_tiles"].tolist()
              for n0 in range(0, cnt, _cabi.I8_BN)]
    naive = sum(int(chunks(pl["knots"][a + c - 1] + 1)) for a, c in per_64)
    assert int(chunks(tiles[:, 3]).sum()) < naive
