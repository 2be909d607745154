"""sharding.EntityRouter (host side of entity-table mode on X-slabs): spawns go to the owner of their column, moves and despawns
to the id's current owner, hand-off lists become adoption batches.  CPU only."""
import numpy as np

from channeld_b200.sharding import EntityRouter, owner_of_column, slab_columns


def test_router_follows_spawns_moves_despawns_and_handoffs():
    world, cols, offx, w = 3, 10, -500.0, 100.0  # rank 0: columns 0-2, rank 1: 3-5, rank 2: 6-9
    assert [slab_columns(cols, world, r) for r in range(world)] == [(0, 3), (3, 6), (6, 10)]
    r = EntityRouter(world, cols, offx, w)
    ids = np.array([1, 2, 3, 4, 5, 6], np.uint32)
    x = np.array([-450.0, -150.0, 150.0, 499.0, -9000.0, 9000.0])  # columns 0, 3, 6, 9; out of the world left and right
    z = np.arange(6, dtype=np.float64)
    b = r.spawn(ids, x, z)
    assert [bb[0].tolist() for bb in b] == [[1, 5], [2], [3, 4, 6]]
    assert b[2][1].tolist() == [150.0, 499.0, 9000.0] and b[2][2].tolist() == [2.0, 3.0, 5.0]
    # a second spawn of a live id goes to its owner, whatever the position (the engine reports the duplicate there)
    b = r.spawn([2, 7], [450.0, 1e-9], [0.0, 0.0])
    assert [bb[0].tolist() for bb in b] == [[], [2, 7], []]
    assert r.owner[2] == 1 and r.owner[7] == 1
    # moves go to the current owner even when they cross a slab border; unknown ids go nowhere
    b = r.move([1, 3, 99], np.array([450.0, -450.0, 0.0], np.float32), [0.0, 0.0, 0.0])
    assert [bb[0].tolist() for bb in b] == [[1], [], [3]]
    assert b[0][1].dtype == np.float32
    # hand-offs: rank 0 gives 1 to rank 2, rank 2 gives 3 to rank 0; positions pass through unchanged
    xa = np.nextafter(450.0, 1e9)
    lists = [(np.array([1], np.uint32), np.array([2], np.uint32), np.array([xa]), np.array([0.25])),
             (np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(0), np.zeros(0)),
             (np.array([3], np.uint32), np.array([0], np.uint32), np.array([-450.0]), np.array([-0.0]))]
    a = r.handoff(lists)
    assert [aa[0].tolist() for aa in a] == [[3], [], [1]]
    assert a[2][1][0] == xa and a[2][2][0] == 0.25 and np.signbit(a[0][2][0])
    assert r.owner[1] == 2 and r.owner[3] == 0
    b = r.move([1, 3], [450.0, -450.0], [0.0, 0.0])
    assert [bb[0].tolist() for bb in b] == [[3], [], [1]]
    # despawns go to the owner and leave the map
    d = r.despawn([1, 5, 42])
    assert [dd.tolist() for dd in d] == [[5], [], [1]]
    assert 1 not in r.owner and 5 not in r.owner
    assert [bb[0].tolist() for bb in r.move([1], [0.0], [0.0])] == [[], [], []]


def test_router_spawn_owner_is_the_owner_of_the_clamped_column():
    world, cols, offx, w = 4, 7, 0.0, 10.0
    r = EntityRouter(world, cols, offx, w)
    x = np.array([-1e30, -0.5, 0.0, 9.999, 35.0, 69.99, 70.0, 1e30, np.nan])
    want_col = np.array([0, 0, 0, 0, 3, 6, 6, 6, 0])
    np.testing.assert_array_equal(r.owner_of_x(x), owner_of_column(want_col, cols, world))
