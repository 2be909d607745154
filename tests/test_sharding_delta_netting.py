"""The host-side netting of a migrated connection's id-mode visible deltas (sharding.net_migrant_delta).  No GPU."""
import numpy as np

from channeld_b200 import sharding


def test_net_migrant_delta_is_the_set_difference_of_the_connection():
    before = [7, 3, 12, 40, 5]          # what the connection saw on rank A (A's leave list for its old slot)
    after = [12, 9, 5, 41, 7, 100]      # what it sees on rank B (B's enter list for its new slot)
    enter, leave = sharding.net_migrant_delta(before, after)
    assert enter.dtype == np.uint32 and leave.dtype == np.uint32
    assert enter.tolist() == [9, 41, 100]  # B's order is kept
    assert leave.tolist() == [3, 40]       # A's order is kept
    assert set(enter) == set(after) - set(before) and set(leave) == set(before) - set(after)


def test_net_migrant_delta_edges():
    e, l = sharding.net_migrant_delta([], [4, 2])
    assert e.tolist() == [4, 2] and l.tolist() == []
    e, l = sharding.net_migrant_delta([4, 2], [])
    assert e.tolist() == [] and l.tolist() == [4, 2]
    e, l = sharding.net_migrant_delta(np.array([1, 2, 3], np.uint32), np.array([3, 2, 1], np.uint32))
    assert len(e) == 0 and len(l) == 0
    # a connection that did not migrate: its enter and leave lists are disjoint, netting them changes nothing
    e, l = sharding.net_migrant_delta([8, 6], [1, 0xFFFFFFFE])
    assert e.tolist() == [1, 0xFFFFFFFE] and l.tolist() == [8, 6]
