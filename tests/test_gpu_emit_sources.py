"""The emit kernels' reads of the cell CSR's sorted entity array, bit-exact against the oracle.

A 16-byte output chunk whose source starts m != 0 entries into an aligned 16-byte chunk takes the rest of its entries from
the next aligned chunk.  These layouts put such chunks on every path that does it: the general-tile kernel next to the CTA
kernel (at least 1 024 entities per cell, a small world), the warp-tile kernel (fewer than 1 024 entities per cell), and in
both the per-entry search of tiles with more pairs than their shared-memory table holds and the last entries of the array,
whose next aligned chunk lies past N.  The test cannot see which kernel ran, so each layout checks, in Python, that it sits on
the intended side of the host's kernel choice and that the tiles it produces hold the cases named above.
Run on an H100:  python -m pytest tests -m gpu
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S0 = 65536
EMIT_TILE, EMIT_SMEM_PAIRS = 2048, 256  # CTA kernels (chd_types.cuh)
EMIT_WARP_TILE, EMIT_WARP_SMEM_PAIRS, EMIT_WARP_ROW = 1024, 64, 128  # warp kernel: 32 lanes x 16 bytes per row


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
    ns.capi, ns.engine, ns.synth = capi, engine, synth
    ns.l2_bytes = torch.cuda.get_device_properties(0).L2_cache_size
    return ns


def _oracle_grid(wc):
    from tests._oracle import make_grid

    return make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)


def _world(oracle, wc, counts, seed):
    """Entities of the 2x2 grid: counts[k] of them inside the k-th cell in CSR order, none out of the world, so the last cell
    ends at the end of the sorted array.  Returns the positions and the cell centres in CSR order."""
    og = _oracle_grid(wc)
    centres = [(wc.offx + (c + 0.5) * wc.w, wc.offz + (r + 0.5) * wc.h) for r in range(wc.rows) for c in range(wc.cols)]
    ids = oracle.cell_of(og, np.array([c[0] for c in centres]), np.array([c[1] for c in centres]))
    centres = [centres[k] for k in np.argsort(ids)]
    rng = np.random.default_rng(seed)
    xs = [cx + rng.uniform(-0.4, 0.4, n) * wc.w for (cx, _), n in zip(centres, counts)]
    zs = [cz + rng.uniform(-0.4, 0.4, n) * wc.h for (_, cz), n in zip(centres, counts)]
    perm = rng.permutation(sum(counts))
    return np.concatenate(xs)[perm], np.concatenate(zs)[perm], centres


def _subscribers(centres, n_mixed, n_tiny, tiny_cells, seed):
    """r = 50 spheres: n_mixed subscribers that each see one cell, two adjacent cells or all four (random), then n_tiny that
    each see one of `tiny_cells` only, then n_mixed more of the first kind."""
    views = [centres[k] for k in range(4)]
    views += [((a[0] + b[0]) / 2, (a[1] + b[1]) / 2) for i, a in enumerate(centres) for b in centres[i + 1:] if a[0] == b[0] or a[1] == b[1]]
    views.append((sum(c[0] for c in centres) / 4, sum(c[1] for c in centres) / 4))
    rng = np.random.default_rng(seed)
    pick = list(rng.integers(0, len(views), n_mixed)) + [tiny_cells[i % len(tiny_cells)] for i in range(n_tiny)] + list(rng.integers(0, len(views), n_mixed))
    cx = np.array([views[k][0] for k in pick])
    cz = np.array([views[k][1] for k in pick])
    return cx, cz, np.full(len(pick), 50.0)


def _check_layout(want, cs, warp):
    """What the visible lists of `want` make the emit kernels do, from the output segments (one per non-empty pair):
    tiles with more than two segments, a tile with more pairs than the shared-memory table, whole chunks at every source
    residue mod 4, a whole chunk with m != 0 whose next aligned chunk lies past N, and (warp tiles) a segment that continues
    from lane 31 of one row into lane 0 of the next with m != 0."""
    tile, smem_pairs = (EMIT_WARP_TILE, EMIT_WARP_SMEM_PAIRS) if warp else (EMIT_TILE, EMIT_SMEM_PAIRS)
    n = int(cs[-1])
    cell = want["pair_cell"].astype(np.int64) - S0
    length = np.diff(cs.astype(np.int64))[cell]
    ob = np.concatenate([[0], np.cumsum(length)[:-1]])[length > 0]
    sb = cs.astype(np.int64)[cell][length > 0]
    length = length[length > 0]
    oe = ob + length
    n_tiles = (int(oe[-1]) + tile - 1) // tile
    per_tile = np.zeros(n_tiles, np.int64)
    for t0, t1 in zip(ob // tile, (oe - 1) // tile):
        per_tile[t0:t1 + 1] += 1
    assert per_tile.max() > smem_pairs
    # the chunk path: tiles whose segment table fits in shared memory (on CTA tiles the general kernel's, more than two segments)
    chunk_tile = per_tile <= smem_pairs
    if not warp:
        chunk_tile &= per_tile > 2
    assert (chunk_tile & (per_tile > 2)).sum() >= 4
    m_seen, past_end, row_cross = set(), False, False
    for b, s, e in zip(ob, sb, oe):
        for t in range(b // tile, (e - 1) // tile + 1):
            if not chunk_tile[t]:
                continue
            lo, hi = max(b, t * tile), min(e, (t + 1) * tile)
            first, last = -(-lo // 4) * 4, hi // 4 * 4 - 4  # whole chunks of this segment inside tile t
            if first > last:
                continue
            m = (s - b) % 4
            m_seen.add(m)
            src_last = s + (last - b)
            past_end |= m != 0 and (src_last - m) + 8 > n
            row_cross |= m != 0 and -(-(first + 4) // EMIT_WARP_ROW) * EMIT_WARP_ROW <= last  # whole chunks at r - 4 and r
    assert m_seen == {0, 1, 2, 3}
    assert past_end
    if warp:
        assert row_cross


# (entities per cell in CSR order: the last cell is the big one and N % 4 != 0), the CSR index of the 2- and 3-entity cells
LAYOUTS = {
    "cta": ([2, 3, 7, 5001], [0, 1]),
    "warp": ([2, 3, 7, 901], [0, 1]),
}


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_emit_sources_layouts(chd, oracle, name):
    counts, tiny = LAYOUTS[name]
    warp = name == "warp"
    wc = chd.synth.CONFIGS["2x2"]
    og = _oracle_grid(wc)
    ex, ez, centres = _world(oracle, wc, counts, seed=11)
    n = len(ex)
    assert n % 4 != 0
    # which side of emit_uses_cta_tiles (chd_tick.cu) the layout is on: mean entities per cell >= EMIT_TILE / 2 and 16 N <= L2 / 2
    assert (n // wc.cells >= EMIT_TILE // 2) == (not warp) and n * 16 <= chd.l2_bytes // 2
    cx, cz, r = _subscribers(centres, 150, 700, tiny, seed=12)
    want = oracle.sphere_tick(og, ex, ez, cx, cz, r)
    cs = np.concatenate([[0], np.cumsum(counts)])
    _check_layout(want, cs, warp)
    e = chd.engine.Engine(wc.cfg(), n, len(cx), max_visible=int(len(want["vis_entity"]) + 4096))
    e.set_entities(ex, ez)
    e.set_subscribers(np.arange(1, len(cx) + 1, dtype=np.uint32))
    batch, keep = chd.engine.make_batch(len(cx), sub=None, sphere=(cx, cz, r))
    for tick in range(3):  # direct launches, then the replayed graphs
        s = e.tick(batch, (tick + 1) * 33_000_000, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
        assert s.overflow == 0 and s.n_visible == len(want["vis_entity"])
        voff, vis = e.get_visible()
        np.testing.assert_array_equal(voff, want["vis_off"])
        np.testing.assert_array_equal(vis, want["vis_entity"])
    np.testing.assert_array_equal(e.get_cells()[0], cs)
    e.close()
