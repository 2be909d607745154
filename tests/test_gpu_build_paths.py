"""The entity build (cell assignment + stable radix sort of entity indices by cell + cell CSR) at its switch points, checked
exactly against a stable sort of the oracle's GetChannelId.

Keys are cells plus one out-of-world key C, so the build sorts C + 1 keys:
  C = 255         256 keys  -> 1 pass, 256 bins (the out-of-world key is the last bin)
  C = 256, 300    -> 1 pass, 1024 bins
  C = 1023        1024 keys -> 1 pass, 1024 bins (the out-of-world key is the last bin)
  C = 1024, 1025  -> 2 passes + cell_bounds_kernel
N: empty, one entity, either side of a BUILD_TILE (2048) and either side of the shared-memory reordered scatter (N > 2^21).
Single-pass builds run as two halves (histogram + CSR offsets, then the scatter); every build runs with and without CUDA graphs,
six times in a row on one engine, so the handover list (entities whose cell changed since the previous build) is checked too.
Run on an H100:  python -m pytest tests/test_gpu_build_paths.py -m gpu
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S0 = 65536
CELL = 10.0
GRIDS = {255: (17, 15), 256: (16, 16), 300: (20, 15), 1023: (33, 31), 1024: (32, 32), 1025: (41, 25)}
COUNTS = [0, 1, 2047, 2048, 2049, 1 << 21, (1 << 21) + 1]


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.capi, ns.engine = capi, engine
    return ns


def _positions(rng, cols, rows, n):
    """The sequence of position sets one engine builds: uniform, the same moved, all in one cell, all outside the world, a
    heavy last cell (with some outside the world), uniform again."""
    W, H = cols * CELL, rows * CELL

    def uniform():
        return rng.random(n) * W, rng.random(n) * H

    def in_cell(k, x, z, m):
        x[m] = (k % cols + rng.random(m.sum())) * CELL
        z[m] = (k // cols + rng.random(m.sum())) * CELL
        return x, z

    x0, z0 = uniform()
    moved = (np.clip(x0 + rng.uniform(-CELL, CELL, n), 0, W - 1e-6), np.clip(z0 + rng.uniform(-CELL, CELL, n), 0, H - 1e-6))
    one = in_cell(int(rng.integers(0, cols * rows)), np.zeros(n), np.zeros(n), np.ones(n, bool))
    out = (-1.0 - rng.random(n) * W, rng.random(n) * H)
    hx, hz = uniform()
    hx, hz = in_cell(cols * rows - 1, hx, hz, rng.random(n) < 0.7)
    far = rng.random(n) < 0.05
    hx[far] = W + rng.random(far.sum())  # x == W is outside the world too
    hx[rng.random(n) < 0.01] = W
    return [(x0, z0), moved, one, out, (hx, hz), uniform()]


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("cells", list(GRIDS))
def test_build_paths_exact(chd, oracle, cells, n):
    from tests._oracle import make_grid

    cols, rows = GRIDS[cells]
    assert cols * rows == cells
    og = make_grid(0.0, 0.0, CELL, CELL, cols, rows)
    sets = _positions(np.random.default_rng(cells * 31 + n), cols, rows, n)
    want = []
    for x, z in sets:
        ids = oracle.cell_of(og, x, z)
        valid = np.nonzero(ids)[0]
        want.append((ids, valid[np.argsort(ids[valid], kind="stable")].astype(np.uint32),
                     np.concatenate([[0], np.cumsum(np.bincount(ids[valid] - S0, minlength=cells))]).astype(np.uint32)))
    for graphs in (True, False):
        e = chd.engine.Engine(chd.engine.grid_cfg(0.0, 0.0, CELL, CELL, cols, rows), max(n, 1), 1)
        e.enable_graphs(graphs)
        for k, ((x, z), (ids, order, cs_want)) in enumerate(zip(sets, want)):
            e.set_entities(x, z)
            e.build()
            s = e.summary()
            assert s.n_entities_in_world == len(order), (graphs, k)
            cs, se = e.get_cells()
            np.testing.assert_array_equal(cs, cs_want, err_msg="cell_start, build %d graphs=%s" % (k, graphs))
            np.testing.assert_array_equal(se, order, err_msg="sorted entities, build %d graphs=%s" % (k, graphs))
            # handover: the entities whose GetChannelId changed since the previous build (0 = outside the world)
            if k == 0:
                assert s.n_handover == 0
                continue
            prev = want[k - 1][0]
            moved = np.nonzero(prev != ids)[0]
            assert s.n_handover == len(moved), (graphs, k)
            ent, src, dst = e.get_handover(s.n_handover)
            o = np.argsort(ent)
            np.testing.assert_array_equal(ent[o], moved.astype(np.uint32))
            np.testing.assert_array_equal(src[o], prev[moved])
            np.testing.assert_array_equal(dst[o], ids[moved])
        e.close()
