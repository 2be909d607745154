"""The emit kernels copy the visible list tile by tile (chd_emit.cuh); whatever order the tiles are taken in, every tile must be
copied exactly once to its own place.  Before each checked tick the whole visible list is filled with a sentinel, so a tile
that no CTA or warp took cannot pass by leaving the previous tick's bytes in place; then every subscriber's list is compared
with the oracle.

Two worlds, one on each side of the host's kernel choice (emit_uses_cta_tiles): CTA tiles, where each cell is shared by
hundreds of pairs, and warp tiles.  Both hold empty cells and entities outside the world.  Each runs seven ticks: four at one
set of radii (direct launches, then the replayed graphs), two at radii that make V several times larger (the CTA grid, sized
from the previous tick's V, is too small and its CTAs loop over the remaining tiles), and one back at the first radii (more
CTAs than tiles).
Run on an H100:  python -m pytest tests -m gpu
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EMIT_TILE = 2048  # chd_types.cuh
SENTINEL = 0xDEADBEEF


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine, synth

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.torch, ns.capi, ns.engine, ns.synth = torch, capi, engine, synth
    ns.l2_bytes = torch.cuda.get_device_properties(0).L2_cache_size
    return ns


class _DeviceArray:
    """A device pointer as torch sees it (__cuda_array_interface__), without a copy."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def _fill_visible(chd, e):
    ptr, n = e.device_view(chd.capi.VIEW_VIS_ENTITY)
    t = chd.torch.as_tensor(_DeviceArray(ptr, n), device="cuda")
    t.fill_(SENTINEL - (1 << 32))  # (the same 32 bits as an int32)
    chd.torch.cuda.synchronize()


def _oracle_grid(wc):
    from tests._oracle import make_grid

    return make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)


# (grid: offset, cell size, cols, rows), entities, subscribers, radii of the first ticks, factor of the large ticks, cells to empty
WORLDS = {
    "cta": ((-4000.0, 2000.0, 4, 4), 24_000, 2_000, (50.0, 1500.0), 4.0, [(1, 2), (3, 0)]),
    "warp": ((-800.0, 100.0, 16, 16), 38_400, 4_000, (20.0, 120.0), 4.0, [(0, 0), (5, 7), (6, 7), (15, 15)]),
}


@pytest.mark.parametrize("name", sorted(WORLDS))
def test_emit_cell_order_every_list(chd, oracle, name):
    (off, size, cols, rows), n, n_sub, (r_lo, r_hi), grow, empty = WORLDS[name]
    wc = chd.synth.WorldConfig("emit-order-" + name, off, off, size, size, cols, rows, 1, 1, n, n_sub, r_lo, 31)
    ex, ez = chd.synth.entities(wc)
    col = np.floor((ex - wc.offx) / wc.w).astype(np.int64)
    row = np.floor((ez - wc.offz) / wc.h).astype(np.int64)
    gone = np.zeros(n, bool)
    for c, r in empty:
        gone |= (col == c) & (row == r)
    # the entities of the emptied cells leave the world (left of it, or below it)
    ex[gone & (np.arange(n) % 2 == 0)] = wc.offx - 7.0
    ez[gone & (np.arange(n) % 2 == 1)] = wc.offz - 3.0
    assert gone.sum() > 0
    # which side of emit_uses_cta_tiles (chd_tick.cu) the world is on: mean entities per cell >= EMIT_TILE / 2
    assert (n // wc.cells >= EMIT_TILE // 2) == (name == "cta") and n * 16 <= chd.l2_bytes // 2

    rng = np.random.default_rng(41)
    inside = np.nonzero(~gone)[0]
    stand = inside[rng.integers(0, len(inside), n_sub)]
    cx, cz = ex[stand].copy(), ez[stand].copy()
    r_small = rng.uniform(r_lo, r_hi, n_sub)
    phases = [r_small] * 4 + [r_small * grow] * 2 + [r_small]
    og = _oracle_grid(wc)
    wants = {}
    for k, r in enumerate(phases):
        key = 0 if k < 4 or k == 6 else 1
        if key not in wants:
            wants[key] = oracle.sphere_tick(og, ex, ez, cx, cz, r)
    v_small, v_large = len(wants[0]["vis_entity"]), len(wants[1]["vis_entity"])
    assert v_large > 3 * v_small
    if name == "cta":  # hundreds of pairs share each non-empty cell
        pairs_per_cell = np.bincount(wants[0]["pair_cell"] - wants[0]["pair_cell"].min())
        assert np.median(pairs_per_cell[pairs_per_cell > 0]) >= 200

    e = chd.engine.Engine(wc.cfg(), n, n_sub, max_visible=v_large + 4096, max_pairs=len(wants[1]["pair_cell"]) + 4096,
                          max_window_cells=4 * len(wants[1]["pair_cell"]) + 4096)
    e.set_entities(ex, ez)
    e.set_subscribers(np.arange(1, n_sub + 1, dtype=np.uint32))
    for tick, r in enumerate(phases):
        want = wants[0 if tick < 4 or tick == 6 else 1]
        batch, keep = chd.engine.make_batch(n_sub, sub=None, sphere=(cx, cz, r))
        _fill_visible(chd, e)
        s = e.tick(batch, (tick + 1) * 33_000_000, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
        assert s.overflow == 0 and s.n_visible == len(want["vis_entity"])
        voff, vis = e.get_visible()
        np.testing.assert_array_equal(voff, want["vis_off"])
        assert not (vis == SENTINEL).any(), "tick %d: %d entries never written" % (tick, int((vis == SENTINEL).sum()))
        np.testing.assert_array_equal(vis, want["vis_entity"])  # every subscriber's list (the offsets are equal)
    e.close()
