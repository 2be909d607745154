"""Followers on sharded entity-table engines: a follower lives on the rank that owns its entity, its query is generated there from
the exact position, a query that would reach columns the slab does not serve is reported as CHD_FOLLOW_OUTSIDE_SLAB, and the
follower moves with its entity (sharding.FollowerRegistry).  Slab engines on one device are fed through sharding.EntityRouter and
checked every tick against one whole-world table engine with the same bindings.
Run on an H100:  python -m pytest tests/test_gpu_sharded_follow.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_follow import assert_same, refused, snapshot
from tests.test_gpu_sharded_table import _vis_sets

pytestmark = pytest.mark.gpu

MS = 1_000_000
TICK = 33 * MS
SPHERE, BOX, CONE = 4, 2, 8
COLS, ROWS, W = 24, 16, 100.0
VIS_FLAGS = 1 | 2  # TICK_BUILD | TICK_EMIT


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine, sharding

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.capi, ns.engine, ns.sharding, ns.torch = capi, engine, sharding, torch
    return ns


def _cfg(chd):
    return chd.engine.grid_cfg(0, 0, W, W, COLS, ROWS)


def _shapes(rng, m):
    """mixed kinds; reach (sph_r, box_ex, cone_r) at most 180, so halo_columns(180) = 2"""
    kind = np.array([SPHERE, BOX, CONE, SPHERE | BOX, SPHERE | CONE, BOX | CONE, SPHERE | BOX | CONE], np.uint8)[np.arange(m) % 7]
    ang = rng.uniform(0, 2 * np.pi, m)
    shape = np.stack([rng.uniform(20, 180, m), rng.uniform(10, 180, m), rng.uniform(10, 120, m), np.cos(ang), np.sin(ang),
                      rng.uniform(0.2, 1.4, m), rng.uniform(30, 180, m)])
    return kind, shape


def _bind(e, slots, ids, kind, shape):
    e.follow_bind(np.asarray(slots, np.uint32), np.asarray(ids, np.uint32), kind=np.asarray(kind, np.uint8), sph_r=shape[0],
                  box=(shape[1], shape[2]), cone=tuple(shape[3:7]))


def _reach_span(x, kind, shape):
    """the column span of a generated query (chd_follow.cuh FollowSlab), before clipping -> (a, b)"""
    a, b = np.inf, -np.inf
    for bit, row in ((SPHERE, 0), (BOX, 1), (CONE, 6)):
        if kind & bit:
            r = shape[row]
            a = min(a, np.floor((x - r - 0.0) / W))
            b = max(b, np.floor((x + r - 0.0) / W))
    return a, b


def _outside(x, kind, shape, lo_col, hi_col, halo):
    """-> 0 inside, -1 leaves the served range on the left, +1 on the right (the clipped span; the world's edges are open)"""
    a, b = _reach_span(x, kind, shape)
    if not (b >= 0 and a < COLS and a <= b):
        return 0
    lo, hi = max(0, lo_col - halo), min(COLS, hi_col + halo)
    if lo > 0 and a < lo:
        return -1
    if hi < COLS and b >= hi:
        return 1
    return 0


class Walk:
    """n entities (ids 1..n) at random places; every tick each one not pinned moves by less than a column in x and z"""

    def __init__(self, n, seed, step=90.0):
        self.rng = np.random.default_rng(seed)
        self.ids = np.arange(1, n + 1, dtype=np.uint32)
        self.x = self.rng.uniform(0, COLS * W, n)
        self.z = self.rng.uniform(0, ROWS * W, n)
        self.pinned = np.zeros(n, bool)
        self.step = step

    def tick(self):
        m = ~self.pinned
        self.x[m] = np.clip(self.x[m] + self.rng.uniform(-self.step, self.step, m.sum()), 0, COLS * W - 1e-6)
        self.z[m] = np.clip(self.z[m] + self.rng.uniform(-self.step, self.step, m.sum()), 0, ROWS * W - 1e-6)
        return self.ids[m], self.x[m].copy(), self.z[m].copy()


class Slabs:
    """`world` table-mode slab engines on one device, joined by host-side border concatenation (no communicator), with the entity
    router and the follower registry every process of a sharded host keeps.  A follower moves as remove on the giver, then add +
    bind on the receiver."""

    def __init__(self, chd, world, halo, n, max_subs):
        import torch

        self.chd, self.world, self.halo, self.n = chd, world, halo, n
        self.cap = n
        self.engines = []
        for r in range(world):
            e = chd.engine.Engine(_cfg(chd), 2 * n + n * world + 16, max_subs, max_visible=1 << 24)
            e.set_slab(*chd.sharding.slab_columns(COLS, world, r), halo)  # the slab first, then the table
            e.entity_table_init()
            self.engines.append(e)
        self.recs = [torch.empty(2 * self.cap, dtype=torch.int32, device="cuda") for _ in range(world)]
        self.router = chd.sharding.EntityRouter(world, COLS, 0.0, W)
        self.reg = chd.sharding.FollowerRegistry(world)
        self.vacated = [[] for _ in range(world)]

    def spawn(self, ids, x, z):
        for e, b in zip(self.engines, self.router.spawn(ids, x, z)):
            if len(b[0]):
                assert (e.spawn_entities(*b) == 0).all()

    def move(self, ids, x, z):
        for e, b in zip(self.engines, self.router.move(ids, x, z)):
            if len(b[0]):
                e.move_entities(*b)

    def place(self):
        """the registry's plan applied -> connections that changed rank this tick"""
        for r, v in enumerate(self.vacated):  # the slots the previous tick's emigrants left are free now
            self.reg.slots.release(r, v)
        arrivals, out_lists, in_calls, vacated, binds = self.reg.plan(self.router)
        for r, v in enumerate(vacated):
            if v:
                self.engines[r].remove_subscribers(v)  # (unbinds)
        moved = set()
        for dst, src, first, pairs in in_calls:
            self.engines[dst].add_subscribers([s for _, s in pairs], [c for c, _ in pairs])
            moved |= {c for c, _ in pairs}
        for r, a in enumerate(arrivals):
            if a:
                self.engines[r].add_subscribers([s for _, s in a], [c for c, _ in a])
        for r, b in enumerate(binds):
            if len(b["conn"]):
                _bind(self.engines[r], b["slot"], b["entity"], b["kind"], b["shape"])
        self.vacated = vacated
        return moved

    def tick(self, t_ns, mode):
        import torch

        for r, e in enumerate(self.engines):
            assert e.export_border(self.recs[r], self.cap) <= self.cap
        torch.cuda.synchronize()
        gathered = torch.cat(self.recs)
        for r, e in enumerate(self.engines):
            e.import_halo(gathered, self.cap * self.world, r * self.cap, self.cap)
            e.build()
            e.follow_queries(mode)
            e.update_interest(None, t_ns)
            e.emit_visible()
            s = e.summary()
            assert s.overflow == 0
        torch.cuda.synchronize()
        del gathered

    def handoff(self):
        """every rank's hand-off list adopted by its destination -> the ids handed off"""
        lists = []
        for r, e in enumerate(self.engines):
            ids, dst, x, z = e.handoff_entities()
            owner = self.chd.sharding.owner_of_column(self.chd.sharding.column_of(x, 0.0, W, COLS), COLS, self.world)
            assert not (owner == r).any()
            lists.append((ids, owner, x, z))
        for r, (ids, x, z) in enumerate(self.router.handoff(lists)):
            if len(ids):
                assert (self.engines[r].spawn_entities(ids, x, z) == 0).all()
        return [int(i) for l in lists for i in l[0].tolist()]

    def close(self):
        for e in self.engines:
            e.close()


def _results(e):
    """slot -> dict(vis, pairs, follow) of every slot of e"""
    vis = _vis_sets(*e.get_visible()) if e.n_slots else []
    p = e.get_pairs()
    f = e.get_follow()
    fol = {int(s): (int(f["entity"][k]), int(f["status"][k]), float(f["cx"][k]), float(f["cz"][k])) for k, s in enumerate(f["slot"])}
    out = {}
    for s in range(e.n_slots):
        a, b = int(p["off"][s]), int(p["off"][s + 1])
        out[s] = dict(vis=vis[s], pairs=list(zip(p["channel"][a:b].tolist(), p["dist"][a:b].tolist(), p["interval"][a:b].tolist())),
                      follow=fol.get(s))
    return out


def _world_setup(chd, world, halo_extra, mode, seed, n=6000, F=480, edge=False):
    rng = np.random.default_rng(seed)
    walk = Walk(n, seed)
    fol_ids = rng.choice(walk.ids, F, replace=False)
    kind, shape = _shapes(rng, F)
    if edge:  # the first followed entities of each side stand at the world's edges, with the largest sphere
        for j, x in enumerate((0.5, 1.0, COLS * W - 0.5, COLS * W - 1.0)):
            walk.x[fol_ids[j] - 1] = x
            walk.pinned[fol_ids[j] - 1] = True
            kind[j], shape[0, j] = SPHERE, 180.0
    halo = chd.sharding.halo_columns(180.0, W) + halo_extra
    sl = Slabs(chd, world, halo, n, F)
    whole = chd.engine.Engine(_cfg(chd), 2 * n, F, max_visible=1 << 24)
    whole.entity_table_init()
    whole.set_subscribers(np.arange(1, F + 1, dtype=np.uint32))  # connection c = slot c - 1
    assert (whole.spawn_entities(walk.ids, walk.x, walk.z) == 0).all()
    sl.spawn(walk.ids, walk.x, walk.z)
    _bind(whole, np.arange(F), fol_ids, kind, shape)
    for j in range(F):
        sl.reg.follow(j + 1, int(fol_ids[j]), int(kind[j]), shape[:, j])
    return walk, fol_ids, kind, shape, halo, sl, whole


# ------------------------------------------------------------------------------------------------- 1. slabs, building blocks
@pytest.mark.parametrize("world", [2, 3])
def test_followers_on_slabs_through_the_building_blocks(chd, world):
    """Every subscriber follows an entity (mixed shapes); the entities walk across slab borders; halo = halo_columns(reach) + 1.
    Every tick, per connection: the visible set, the pairs (cell, dist, interval) and the follower's status equal the whole world's,
    and so does its chd_get_follow entry except on the tick the connection moves to another rank.  Followed entities are handed
    off, and no follower is ever outside its slab."""
    capi = chd.capi
    walk, fol_ids, kind, shape, halo, sl, whole = _world_setup(chd, world, 1, capi.FOLLOW_MOVED, 40 + world)
    F = len(fol_ids)
    handed_followed = moved_total = 0
    for t in range(8):
        if t:
            mv = walk.tick()
            whole.move_entities(*mv)
            sl.move(*mv)
        moved = sl.place()
        moved_total += len(moved)
        whole.follow_queries(capi.FOLLOW_MOVED)
        sw = whole.tick(None, (t + 1) * TICK, VIS_FLAGS | capi.TICK_FOLLOW)
        assert sw.overflow == 0
        sl.tick((t + 1) * TICK, capi.FOLLOW_MOVED)
        wr = _results(whole)
        per = [_results(e) for e in sl.engines]
        for c in range(1, F + 1):
            got, want = per[sl.reg.owner_of(c)][sl.reg.slots.slot[c]], wr[c - 1]
            assert got["vis"] == want["vis"], (t, c)
            assert got["pairs"] == want["pairs"], (t, c)
            assert got["follow"][1] != capi.FOLLOW_OUTSIDE_SLAB, (t, c)
            if c not in moved:
                assert got["follow"] == want["follow"], (t, c)
        handed = set(sl.handoff())
        handed_followed += len(handed & set(fol_ids.tolist()))
    assert handed_followed > 0 and moved_total > 0, (handed_followed, moved_total)
    sl.close()
    whole.close()


# ------------------------------------------------------------------------------------------------- 2. minimal halo
def test_minimal_halo_reports_outside_slab_exactly_where_the_span_leaves_the_served_range(chd):
    """halo = halo_columns(reach): on the tick an entity crosses into a neighbour's slab, its old owner generates the query centred in
    the neighbour's column, and a follower whose clipped column span (numpy, same formula) leaves the served range gets
    CHD_FOLLOW_OUTSIDE_SLAB, with its pairs unchanged that tick.  Every other follower equals the whole world (FOLLOW_ALL), the
    followers at the world's edges included.  Both sides of a slab are covered."""
    capi, world = chd.capi, 3
    walk, fol_ids, kind, shape, halo, sl, whole = _world_setup(chd, world, 0, capi.FOLLOW_ALL, 77, edge=True)
    F = len(fol_ids)
    slabs = [chd.sharding.slab_columns(COLS, world, r) for r in range(world)]
    prev = {}
    sides = {-1: 0, 1: 0}
    for t in range(8):
        if t:
            mv = walk.tick()
            whole.move_entities(*mv)
            sl.move(*mv)
        moved = sl.place()
        whole.follow_queries(capi.FOLLOW_ALL)
        assert whole.tick(None, (t + 1) * TICK, VIS_FLAGS | capi.TICK_FOLLOW).overflow == 0
        sl.tick((t + 1) * TICK, capi.FOLLOW_ALL)
        wr = _results(whole)
        per = [_results(e) for e in sl.engines]
        for c in range(1, F + 1):
            r = sl.reg.owner_of(c)
            got, want = per[r][sl.reg.slots.slot[c]], wr[c - 1]
            x = walk.x[fol_ids[c - 1] - 1]
            side = _outside(x, int(kind[c - 1]), shape[:, c - 1], slabs[r][0], slabs[r][1], halo)
            if side:
                sides[side] += 1
                assert got["follow"][1] == capi.FOLLOW_OUTSIDE_SLAB, (t, c, x, r)
                assert got["pairs"] == ([] if c in moved else prev[c]), (t, c)  # (a slot that just arrived has none yet)
            else:
                assert got["follow"][1] != capi.FOLLOW_OUTSIDE_SLAB, (t, c, x, r)
                assert got["vis"] == want["vis"] and got["pairs"] == want["pairs"], (t, c)
                assert got["follow"][:2] == want["follow"][:2], (t, c)
            if c <= 4:  # the followers at the world's edges
                assert side == 0 and got["follow"][1] == capi.Q_OK, (t, c)
            prev[c] = got["pairs"]
        sl.handoff()
    assert sides[-1] > 0 and sides[1] > 0, sides
    sl.close()
    whole.close()


# ------------------------------------------------------------------------------------------------- 3. halo and handed-off ids
def test_a_follower_of_an_id_another_rank_owns_reports_no_entity_and_resumes_when_adopted(chd):
    capi = chd.capi
    sl = Slabs(chd, 2, 2, 64, 8)  # rank 0: columns [0, 12), rank 1: [12, 24)
    a, b = sl.engines
    bg = np.arange(100, 140, dtype=np.uint32)
    sl.spawn(bg, np.linspace(50, 2350, 40), np.full(40, 400.0))
    sl.spawn([1, 3], [1150.0, 1300.0], [420.0, 420.0])  # 1 is rank 0's; 3 is rank 1's and a halo entity of rank 0
    a.add_subscribers([0, 1], [1, 2])
    _bind(a, [0, 1], [1, 3], [SPHERE, SPHERE], np.array([[50.0] * 2] + [[1.0] * 2] * 6))

    def step(t):
        sl.tick(t * TICK, capi.FOLLOW_MOVED)
        f = a.get_follow()
        return {int(s): (int(f["status"][k]), float(f["cx"][k])) for k, s in enumerate(f["slot"])}, f["n_selected"], _results(a)

    f, n_sel, res = step(1)
    assert f[0] == (capi.Q_OK, 1150.0) and f[1][0] == capi.FOLLOW_NO_ENTITY and n_sel == 1
    assert res[0]["pairs"] and not res[1]["pairs"]
    sl.move([1], [1250.0], [420.0])  # into rank 1's column: rank 0 still owns it this tick
    f, n_sel, res = step(2)
    assert f[0] == (capi.Q_OK, 1250.0)
    kept = res[0]["pairs"]
    assert sl.handoff() == [1]
    f, n_sel, res = step(3)  # handed off: a halo id for rank 0 now
    assert f[0] == (capi.FOLLOW_NO_ENTITY, 1250.0) and n_sel == 0 and res[0]["pairs"] == kept
    sl.move([1], [1150.0], [420.0])  # back into rank 0's column, moved by its owner, rank 1
    f, n_sel, res = step(4)
    assert f[0][0] == capi.FOLLOW_NO_ENTITY and res[0]["pairs"] == kept
    assert sl.handoff() == [1]
    f, n_sel, res = step(5)  # adopted: the follower resumes and counts as moved
    assert f[0] == (capi.Q_OK, 1150.0) and n_sel == 1 and res[0]["pairs"] != kept
    f, n_sel, res = step(6)  # nothing moved
    assert f[0] == (capi.FOLLOW_NOT_SELECTED, 1150.0) and n_sel == 0
    sl.close()


# ------------------------------------------------------------------------------------------------- 4. chd_tick_sharded at world one
def _summary_fields(s):
    d = s.as_dict()
    return {k: d[k] for k in ("n_pairs", "n_visible", "n_query_errors", "n_sub_new", "n_unsub", "n_kept", "n_due", "n_handover", "overflow")}


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
@pytest.mark.parametrize("mig", [0, 64], ids=["no-migration", "migration"])
@pytest.mark.parametrize("merged", [False, True], ids=["follow", "merged"])
def test_tick_sharded_with_followers_at_world_one_matches_a_single_engine(chd, graphs, mig, merged):
    """chd_follow_queries(_with) + chd_tick_sharded(NULL, CHD_TICK_FOLLOW) on a one-rank communicator gives what chd_tick gives on a
    single table engine: summary, pairs, diffs and due list (as sets), statuses and follower reports."""
    capi = chd.capi
    n, S, F = 4000, 300, 200
    walk = Walk(n, 9, step=40.0)
    rng = np.random.default_rng(10)
    kind, shape = _shapes(rng, F)
    fol = rng.choice(walk.ids, F, replace=False)
    sh = chd.engine.Engine(_cfg(chd), 3 * n + 16, S, max_visible=1 << 24, max_queries=1024)
    one = chd.engine.Engine(_cfg(chd), 3 * n + 16, S, max_visible=1 << 24, max_queries=1024)
    sh.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, 2, n, migrate_subscribers=mig)
    for e in (sh, one):
        e.enable_graphs(graphs)
        e.entity_table_init()
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        assert (e.spawn_entities(walk.ids, walk.x, walk.z) == 0).all()
        _bind(e, np.arange(F), fol, kind, shape)
    for t in range(6):
        if t:
            mv = walk.tick()
            for e in (sh, one):
                e.move_entities(*mv)
        n_h = 0
        keep = []
        for e in (sh, one):
            if merged:  # the slots that follow nothing send explicit queries, one of them a follower's override
                k = 20 + 7 * t
                sub = np.concatenate([np.arange(F, F + k), [3]]).astype(np.uint32)
                r2 = np.random.default_rng(100 + t)
                batch, kp = chd.engine.make_batch(len(sub), sub=sub, sphere=(r2.uniform(0, 2400, len(sub)), r2.uniform(0, 1600, len(sub)),
                                                                                r2.uniform(30, 150, len(sub))))
                keep.append(kp)
                n_h = len(sub)
                e.follow_queries_with(capi.FOLLOW_MOVED, batch)
            else:
                e.follow_queries(capi.FOLLOW_MOVED)
        s1 = sh.tick_sharded(None, (t + 1) * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        s2 = one.tick(None, (t + 1) * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
        assert _summary_fields(s1) == _summary_fields(s2), t
        a, b = snapshot(sh, s1, vis=False), snapshot(one, s2, vis=False)
        a["summary"], b["summary"] = None, None
        assert_same(a, b, "tick %d" % t)
        assert _vis_sets(*sh.get_visible()) == _vis_sets(*one.get_visible()), t
        L = chd.engine.host_part_size(n_h) + F
        np.testing.assert_array_equal(sh.get_query_status(L), one.get_query_status(L))
        fa, fb = sh.get_follow(), one.get_follow()
        for k in ("slot", "entity", "status", "cx", "cz"):
            np.testing.assert_array_equal(fa[k], fb[k])
        assert fa["n_selected"] == fb["n_selected"] and fa["n_selected"] > 0
    if graphs:
        assert sh.graph_launch_count() > 0
    assert chd.capi.lib().chd_comm_destroy(sh.h) == capi.OK
    sh.close(), one.close()


# ------------------------------------------------------------------------------------------------- 5. chd_migrate_out unbinds
def test_migrate_out_unbinds_the_emigrants(chd):
    capi = chd.capi
    n, S = 500, 16
    walk = Walk(n, 5)
    rng = np.random.default_rng(6)
    kind, shape = _shapes(rng, S)
    e = chd.engine.Engine(_cfg(chd), 3 * n + 16, S)
    e.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, 2, n, migrate_subscribers=8)
    e.entity_table_init()
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    assert (e.spawn_entities(walk.ids, walk.x, walk.z) == 0).all()
    _bind(e, np.arange(S), walk.ids[:S], kind, shape)
    e.follow_queries(capi.FOLLOW_ALL)
    e.tick_sharded(None, TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    assert e.get_follow()["n_selected"] == S
    e.migrate_out([3, 9])
    e.follow_queries(capi.FOLLOW_ALL)
    e.tick_sharded(None, 2 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    f = e.get_follow()
    assert f["n_selected"] == S - 2 and not {3, 9} & set(f["slot"].tolist()) and len(f["slot"]) == S - 2
    p = e.get_pairs()
    assert p["off"][4] == p["off"][3] and p["off"][10] == p["off"][9]  # the emigrants' subscriptions left with them
    # CHD_TICK_FOLLOW needs a generated batch, and takes no host batch
    refused(e, capi.ERR_STATE, "CHD_TICK_FOLLOW without", "chd_tick_sharded", None, 3 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW, None)
    batch, keep = chd.engine.make_batch(1, sub=np.array([0], np.uint32), sphere=(np.array([10.0]), np.array([10.0]), np.array([50.0])))
    e.follow_queries(capi.FOLLOW_ALL)
    refused(e, capi.ERR_INVALID, None, "chd_tick_sharded", C.byref(batch), 3 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW, None)
    e.tick_sharded(None, 3 * TICK, capi.TICK_ALL | capi.TICK_FOLLOW)
    assert chd.capi.lib().chd_comm_destroy(e.h) == capi.OK
    e.close()


# ------------------------------------------------------------------------------------------------- 6. rules
def test_rule_9_admits_table_mode_slabs_only(chd):
    capi = chd.capi
    one = np.array([0], np.uint32)
    r = np.array([10.0])
    fb = capi.FollowBatch()
    keep = [np.array([0], np.uint32), np.array([1], np.uint32), r]
    fb.n, fb.slot, fb.entity, fb.sph_r = 1, capi.ptr(keep[0]), capi.ptr(keep[1]), capi.ptr(keep[2])
    qb, qk = chd.engine.make_batch(1, sub=np.array([1], np.uint32), sphere=(np.array([10.0]), np.array([10.0]), np.array([50.0])))
    # a table-mode slab takes all five calls
    t = chd.engine.Engine(_cfg(chd), 64, 8, max_queries=512)
    t.set_slab(0, 12, 2)
    t.entity_table_init()
    t.set_subscribers(np.arange(1, 9, dtype=np.uint32))
    assert (t.spawn_entities([1], [50.0], [50.0]) == 0).all()
    assert t.L.chd_follow_bind(t.h, C.byref(fb)) == capi.OK
    t.follow_queries(capi.FOLLOW_ALL)
    t.update_interest(None, TICK)
    assert t.get_follow()["status"].tolist() == [capi.Q_OK]
    t.follow_queries_with(capi.FOLLOW_MOVED, qb)
    t.update_interest(None, 2 * TICK)
    assert t.L.chd_follow_unbind(t.h, capi.ptr(one), 1) == capi.OK
    assert len(t.get_follow()["slot"]) == 0
    # index-mode and id-mode slabs refuse every call
    for ids in (False, True):
        s = chd.engine.Engine(_cfg(chd), 64, 8)
        s.set_subscribers(np.arange(1, 9, dtype=np.uint32))
        s.set_slab(0, 12, 2)
        if ids:
            s.set_entity_ids(np.arange(4, dtype=np.uint32))
        refused(s, capi.ERR_STATE, "slab", "chd_follow_bind", C.byref(fb))
        refused(s, capi.ERR_STATE, "slab", "chd_follow_queries", 0)
        refused(s, capi.ERR_STATE, "slab", "chd_follow_queries_with", 0, C.byref(qb))
        refused(s, capi.ERR_STATE, "slab", "chd_follow_unbind", capi.ptr(one), 1)
        refused(s, capi.ERR_STATE, "slab", "chd_get_follow", None, None, None, None, None, 0, None, None)
        s.close()
    # an engine with followers does not become a slab
    f = chd.engine.Engine(_cfg(chd), 64, 8)
    f.set_subscribers(np.arange(1, 9, dtype=np.uint32))
    f.set_entities(np.array([50.0, 60.0]), np.array([50.0, 60.0]))
    assert f.L.chd_follow_bind(f.h, C.byref(fb)) == capi.OK
    refused(f, capi.ERR_STATE, "follow entities", "chd_set_slab", 0, 12, 1)
    refused(f, capi.ERR_STATE, "follow entities", "chd_comm_init", (C.c_uint8 * 128)(), 0, 1, 1, 16, 0, 0)
    for e in (t, f):
        e.close()
