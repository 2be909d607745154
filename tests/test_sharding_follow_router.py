"""sharding.FollowerRegistry: followers live on the rank that owns their entity.  The plan after each tick's hand-offs places new
followers, migrates the ones whose entity changed owner and gives each destination the chd_follow_bind batch of its arrivals; it is
a pure function of the registry and the router, so every process of a multi-rank host computes the same one."""
import numpy as np

from channeld_b200 import sharding

SHAPE = (50.0, 40.0, 30.0, 1.0, 0.0, 0.5, 60.0)


def _registry(order):
    router = sharding.EntityRouter(3, 30, 0.0, 100.0)
    router.spawn(np.arange(1, 11, dtype=np.uint32), np.arange(10) * 300.0 + 5.0, np.zeros(10))
    reg = sharding.FollowerRegistry(3)
    for c in order:
        reg.follow(c, c // 10, 4 | (c & 2), SHAPE)
    return reg, router


def _plain(plan):
    arrivals, out_lists, in_calls, vacated, binds = plan
    b = [{k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in x.items()} for x in binds]
    return arrivals, out_lists, in_calls, vacated, b


def test_followers_live_with_their_entity_and_move_with_it():
    reg, router = _registry([10 * i for i in range(1, 11)] + [110])  # 110 follows entity 11, which does not exist yet
    arrivals, out_lists, in_calls, vacated, binds = reg.plan(router)
    assert not in_calls and all(not o for o in out_lists)
    for c in range(10, 101, 10):
        assert reg.owner_of(c) == router.owner[c // 10]
    assert reg.owner_of(110) is None
    for r in range(3):
        assert [c for c, _ in arrivals[r]] == binds[r]["conn"]
        np.testing.assert_array_equal(binds[r]["slot"], [s for _, s in arrivals[r]])
        np.testing.assert_array_equal(binds[r]["entity"], [c // 10 for c in binds[r]["conn"]])
        assert binds[r]["shape"].shape == (7, len(arrivals[r])) and (binds[r]["shape"][6] == 60.0).all()
    # entity 1 is handed from rank 0 to rank 2, entity 5 from rank 1 to rank 0; entity 11 spawns on rank 1
    before = {c: (reg.owner_of(c), reg.slots.slot[c]) for c in (10, 50)}
    router.handoff([(np.array([5, 1], np.uint32), np.array([0, 2]), [5.0, 2950.0], [0.0, 0.0])])
    router.spawn(np.array([11], np.uint32), [1500.0], [0.0])
    arrivals, out_lists, in_calls, vacated, binds = reg.plan(router)
    assert reg.owner_of(10) == 2 and reg.owner_of(50) == 0 and reg.owner_of(110) == 1
    assert out_lists[before[10][0]] == [10] and vacated[before[10][0]] == [before[10][1]]
    assert out_lists[before[50][0]] == [50] and vacated[before[50][0]] == [before[50][1]]
    moved = {(dst, src): [c for c, _ in pairs] for dst, src, _, pairs in in_calls}
    assert moved == {(2, before[10][0]): [10], (0, before[50][0]): [50]}
    assert binds[2]["conn"] == [10] and binds[0]["conn"] == [50] and binds[1]["conn"] == [110]
    assert binds[2]["slot"].tolist() == [reg.slots.slot[10]] and binds[2]["entity"].tolist() == [1]
    # a re-bind reaches the follower's rank at the next plan, a plan without changes binds nothing
    reg.follow(60, 6, 8, SHAPE)
    arrivals, out_lists, in_calls, vacated, binds = reg.plan(router)
    assert sum(len(b["conn"]) for b in binds) == 1 and binds[reg.owner_of(60)]["kind"].tolist() == [8]
    assert sum(len(b["conn"]) for b in reg.plan(router)[4]) == 0
    assert reg.unfollow(60) == (router.owner[6], binds[router.owner[6]]["slot"][0])
    assert reg.owner_of(60) is None and 60 not in reg.bind


def test_the_plan_is_the_same_in_every_process():
    """Two registries fed the same events in different registration orders make identical plans tick after tick."""
    rng = np.random.default_rng(3)
    conns = [10 * i for i in range(1, 11)]
    a, ra = _registry(conns)
    b, rb = _registry(list(reversed(conns)))
    for t in range(6):
        pa, pb = _plain(a.plan(ra)), _plain(b.plan(rb))
        assert pa == pb, t
        ids = rng.choice(np.arange(1, 11), 3, replace=False).astype(np.uint32)
        dst = rng.integers(0, 3, 3)
        lists = [(ids[dst == r], dst[dst == r], np.zeros(int((dst == r).sum())), np.zeros(int((dst == r).sum()))) for r in range(3)]
        ra.handoff(lists)
        rb.handoff(lists)
    assert a.slots.owner == b.slots.owner and a.slots.slot == b.slots.slot
