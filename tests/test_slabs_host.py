"""The numpy restatements of tests/_slabs.py against hand-worked cases and against a second formulation: an entity is exported when
it left its slab or when another rank serves its column.  CPU only."""
import numpy as np

from channeld_b200 import sharding, synth
from tests import _slabs


def test_export_set_hand_worked():
    def exported(cols, lo, hi, halo):  # own entities: one per column of the slab, in a one-row grid
        cell = np.arange(lo, hi)
        return _slabs.export_set(cell, cell, cols, lo, hi, halo)[0].tolist()

    # two slabs, halo 1: each exports the column next to the other slab, nothing at the world's edges
    assert exported(15, 0, 7, 1) == [6]
    assert exported(15, 7, 15, 1) == [7]
    # a one-column slab with halo 2 between two open edges: its only column; with the left edge closed: still (right is open)
    assert exported(15, 5, 6, 2) == [5]
    assert exported(15, 0, 1, 2) == [0]
    # the middle slab of three on 15 columns, halo 2: two columns on each side, the interior stays
    assert exported(15, 5, 10, 2) == [5, 6, 8, 9]
    # one slab over the whole world: nothing to export
    assert exported(15, 0, 15, 3) == []
    # entities that left the slab are exported wherever they are; entities outside the world never
    g, c = _slabs.export_set(np.array([3, 12, -1, 10]), np.array([100, 101, 102, 103]), 15, 5, 10, 1)
    assert g.tolist() == [100, 101, 103] and c.tolist() == [3, 12, 10]
    # one-column slabs of the 2 x 2 grid: everything in the world goes out
    g, _ = _slabs.export_set(np.array([0, 2, 1, 3, -1]), np.arange(5), 2, 0, 1, 1)
    assert g.tolist() == [0, 1, 2, 3]


def test_export_set_is_what_other_ranks_serve():
    rng = np.random.default_rng(3)
    for cols, world, halo in ((15, 2, 1), (15, 8, 2), (2, 2, 1), (256, 3, 1), (15, 4, 5), (7, 7, 1)):
        slabs = [sharding.slab_columns(cols, world, r) for r in range(world)]
        cell = rng.integers(-1, cols * 3, 4000)
        cell = np.where(cell >= 0, cell, -1)
        gid = np.arange(len(cell))
        for r, (lo, hi) in enumerate(slabs):
            col = cell % cols
            served_elsewhere = np.zeros(len(cell), bool)
            for q, (a, b) in enumerate(slabs):
                if q != r:
                    sa, sb = _slabs.served_columns(cols, a, b, halo)
                    served_elsewhere |= (col >= sa) & (col < sb)
            want = (cell >= 0) & (served_elsewhere | (col < lo) | (col >= hi))
            assert _slabs.export_set(cell, gid, cols, lo, hi, halo)[0].tolist() == gid[want].tolist(), (cols, world, halo, r)


def test_import_set_and_rehome():
    recs = [(np.array([1, 2, 3]), np.array([0, 6, 16])),      # rank 0 on a 15 x 2 grid: cells in columns 0, 6, 1
            (np.array([4, 5, 6]), np.array([7, 22, 14])),     # rank 1: columns 7, 7, 14
            (np.array([7, 8]), np.array([13, 0xFFFFFFFF]))]   # rank 2: column 13 and a padding record
    g, c, src = _slabs.import_set(recs, 1, 15, 30, 5, 10, 1)  # serves columns [4, 11)
    assert g.tolist() == [2] and c.tolist() == [6] and src.tolist() == [0]
    g, c, src = _slabs.import_set(recs, 0, 15, 30, 0, 5, 3)  # serves [0, 8)
    assert g.tolist() == [4, 5] and src.tolist() == [1, 1]
    g, c, src = _slabs.import_set(recs, 2, 15, 30, 10, 15, 4)  # serves [6, 15)
    assert g.tolist() == [2, 4, 5, 6] and src.tolist() == [0, 1, 1, 1]
    gid, dst = _slabs.rehome_set(np.array([4, 5, 9, 10, -1, 30]), np.array([10, 11, 12, 13, 14, 15]), 15, 5, 10, 3)
    assert gid.tolist() == [10, 13, 15] and dst.tolist() == [0, 2, 0]  # (cell 30: column 0 of row 2)


def test_grid_cells_match_the_oracle_at_column_edges(oracle):
    for name in ("benchmark", "2x2", "handover"):
        wc = synth.CONFIGS[name]
        slabs = [sharding.slab_columns(wc.cols, 3 if wc.cols > 2 else 2, r) for r in range(3 if wc.cols > 2 else 2)]
        x, k = _slabs.boundary_xs(wc.offx, wc.w, wc.cols, slabs, 2)
        z = np.full(len(x), wc.offz + 0.5 * wc.h)
        got = _slabs.grid_cells(x, z, wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows)
        from tests._oracle import make_grid

        og = make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)
        ids = oracle.cell_of(og, x, z).astype(np.int64) - og.channel_id_start
        ids = np.where((ids >= 0) & (ids < wc.cells), ids, -1)
        np.testing.assert_array_equal(got, ids)
        # offx + k * w itself is column k (or outside the world at k < 0 and k >= cols)
        mid = np.arange(1, len(x), 3)
        np.testing.assert_array_equal(got[mid], np.where((k[mid] >= 0) & (k[mid] < wc.cols), k[mid], -1))


def test_emit_kernel_side():
    l2 = 50 << 20
    assert _slabs.emit_uses_cta_tiles(1024 * 105, 7, 15, 1024 * 105, l2)
    assert not _slabs.emit_uses_cta_tiles(1023 * 105, 7, 15, 1023 * 105, l2)
    assert _slabs.emit_uses_cta_tiles(1 << 20, 1, 2, (l2 // 2) // 16, l2)
    assert not _slabs.emit_uses_cta_tiles(1 << 20, 1, 2, (l2 // 2) // 16 + 1, l2)
