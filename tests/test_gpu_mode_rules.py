"""The mode rules (DESIGN.md §5): which calls each way of naming entities admits.  Entities are named by index, by global id
(chd_set_entity_ids) or by table id (entity-table mode, chd_entity_table_init); visible deltas by index or by global id (id mode,
chd_reserve_visible_delta_ids).  With them the call-order rules: one query batch per interest update (9) and nothing rewritten
under a begun chd_begin_interest (13).  A matrix: every row is one engine brought into a mode by a set-up, one gated call and the
status it must return.  Rule numbers follow the table in DESIGN.md §5; one test per rule runs its rows and reports every row that breaks.
Run on an H100:  python -m pytest tests/test_gpu_mode_rules.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_rings_scale import _status

pytestmark = pytest.mark.gpu

OK, INVALID, STATE = 0, 1, 4  # capi.OK, capi.ERR_INVALID, capi.ERR_STATE
DELTA_FLAGS = 1 | 2 | 16  # TICK_BUILD | TICK_EMIT | TICK_VISIBLE_DELTA
ID_SPACE = 1 << 10
MS = 1_000_000


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
    ns.L = capi.lib()
    ns.wc = synth.CONFIGS["2x2"]  # 2 x 2 cells of 2000 x 2000, 1000 entities, 256 subscribers
    ns.x, ns.z = synth.entities(ns.wc)
    return ns


X4, Z4 = np.zeros(4), np.zeros(4)
XF, ZF = np.zeros(4, np.float32), np.zeros(4, np.float32)
GID4 = np.arange(4, dtype=np.uint32)
RING_OFF = np.zeros(2 * 2 + 1, np.uint32)  # empty rings of the 2 x 2 world: every cell's range is [0, 0)


def _engine(chd, n=None):
    wc = chd.wc
    return chd.engine.Engine(wc.cfg(), n or wc.n_entities, wc.n_subscribers)


def _world(chd, e):
    """the world's entities and four subscribers at its centre, each seeing every cell"""
    S = 4
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.set_entities(chd.x, chd.z)
    b, keep = chd.engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(np.zeros(S), np.zeros(S), np.full(S, 50.0)))
    e._rules_batch = (b, keep)
    return e


def _batch(chd, e):
    """four subscribers at the world's centre, and the batch of their queries"""
    S = 4
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e._rules_batch = chd.engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(np.zeros(S), np.zeros(S), np.full(S, 50.0)))
    return e


def _table_slab(chd):
    """a table engine made a slab first; its two entities lie in column 0 (borders the slab edge) and column 1 (beyond it)"""
    e = _engine(chd, 64)
    e.set_slab(0, 1, 1)
    e.entity_table_init()  # (rule 4: a slab may come first)
    return e


# ---------------------------------------------------------------------------------------------------------------- set-ups
def _setups():
    def fresh(chd):
        return _engine(chd, 16)

    def table(chd):
        e = _engine(chd, 16)
        e.entity_table_init()
        return e

    def table_spawned_after_build(chd):
        e = table(chd)
        e.reserve_visible_delta(64)
        e.spawn_entities([1], [0.0], [0.0])
        return e

    def table_built(chd):
        e = table_spawned_after_build(chd)
        e.build()
        return e

    def built(chd):
        e = _engine(chd, 16)
        e.set_entities(X4, Z4)
        e.build()
        return e

    def assigned_without_ids(chd):
        e = _engine(chd, 16)
        e.set_entities(X4, Z4)
        assert chd.L.chd_assign_cells(e.h) == OK
        return e

    def slab(chd):
        e = _engine(chd, 16)
        e.set_slab(0, 1, 1)
        return e

    def slab_ids(chd):
        e = slab(chd)
        e.set_entity_ids(GID4)
        return e

    def slab_ids_null(chd):
        e = slab(chd)
        e.set_entity_ids(None)
        return e

    def ids_null(chd):
        e = _engine(chd, 16)
        e.set_entity_ids(None)
        return e

    def slab_assigned(chd):
        e = slab(chd)
        assert chd.L.chd_assign_cells(e.h) == OK
        return e

    def slab_built(chd):
        e = slab(chd)
        e.set_entities(X4, Z4)
        e.build()
        return e

    def slab_delta_ids(chd):
        e = slab(chd)
        e.reserve_visible_delta_ids(64, ID_SPACE)
        return e

    def index_delta(chd):
        e = _engine(chd)
        e.reserve_visible_delta(64)
        return e

    def id_delta(chd):
        e = _engine(chd)
        e.reserve_visible_delta_ids(64, ID_SPACE)
        return e

    # single-GPU index-mode deltas, then the engine is made a slab / given global ids (the multi-GPU flow)
    def index_delta_then_slab(chd):
        e = _world(chd, _engine(chd))
        e.reserve_visible_delta(1024)
        e.set_slab(0, chd.wc.cols, 0)
        e.set_entities(chd.x, chd.z)
        return e

    def index_delta_then_ids(chd):
        e = _world(chd, _engine(chd))
        e.reserve_visible_delta(1024)
        e.set_entity_ids(np.arange(len(chd.x), dtype=np.uint32))
        e.set_entities(chd.x, chd.z)
        return e

    # id-mode deltas without ids for the own entities, then with ids set after the last build, then with a build after them
    def id_delta_without_ids(chd):
        e = _world(chd, _engine(chd))
        e.reserve_visible_delta_ids(1 << 16, chd.wc.n_entities)
        e.set_entities(chd.x, chd.z)
        return e

    def id_delta_without_ids_built(chd):
        e = id_delta_without_ids(chd)
        e.build()
        return e

    def id_delta_ids_after_build(chd):
        e = id_delta_without_ids_built(chd)
        e.set_entity_ids(np.arange(chd.wc.n_entities, dtype=np.uint32))
        return e

    def id_delta_ids_built(chd):
        e = id_delta_ids_after_build(chd)
        e.build()
        e.update_interest(e._rules_batch[0], 0)
        return e

    def table_slab(chd):
        return _table_slab(chd)

    def table_slab_spawned(chd):
        e = _table_slab(chd)
        e.spawn_entities([5, 6], [-1000.0, 1000.0], [-1000.0, -1000.0])
        return e

    # rule 9: followers; slot 0 follows entity 0 (index mode) or table id 1 (entity-table mode)
    def slab_subscribed(chd):
        return _batch(chd, slab(chd))

    def following_index(chd):
        e = _batch(chd, _engine(chd, 16))
        e.set_entities(X4, Z4)
        e.follow_bind([0], [0], sph_r=[50.0])
        return e

    def followed(chd):
        e = chd.engine.Engine(chd.wc.cfg(), 64, chd.wc.n_subscribers, max_queries=512)  # (merged: a host class of 256 and the follower)
        e.entity_table_init()
        e.spawn_entities([1, 2], [0.0, 10.0], [0.0, 10.0])
        _batch(chd, e)
        e.follow_bind([0], [1], sph_r=[50.0])
        return e

    def generated(chd):
        e = followed(chd)
        e.follow_queries()
        return e

    def adopted(chd):
        e = followed(chd)
        e.prefetch_queries(*e._rules_batch)
        e.adopt_prefetched()
        return e

    # rule 12: device rings on one GPU, and on a one-rank communicator (a slab)
    def rings(chd):
        e = _batch(chd, _engine(chd, 16))
        e.set_entities(X4, Z4)
        assert chd.L.chd_rings_init(e.h, 513) == OK
        return e

    def comm_rings(chd):
        e = _engine(chd, 256)  # (room for the halo of a border capacity of 64)
        e.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, 1, 64)
        _batch(chd, e)
        assert chd.L.chd_rings_init(e.h, 513) == OK
        e.set_entities(X4, Z4)
        e.set_entity_ids(GID4)
        return e

    def comm_rings_staged(chd):
        e = comm_rings(chd)
        assert chd.L.chd_rings_append(e.h, chd.capi.ptr(RING_OFF), 0, None, None) == OK
        return e

    fns = [fresh, table, table_spawned_after_build, table_built, built, assigned_without_ids, slab, slab_ids, slab_ids_null, ids_null, slab_assigned,
           slab_built, slab_delta_ids, index_delta, id_delta, index_delta_then_slab, index_delta_then_ids, id_delta_without_ids,
           id_delta_without_ids_built, id_delta_ids_after_build, id_delta_ids_built, table_slab, table_slab_spawned, slab_subscribed,
           following_index, followed, generated, adopted, rings, comm_rings, comm_rings_staged]
    out = {f.__name__: f for f in fns}

    # rule 13: a chd_begin_interest begun with or without the fan-out, and then joined by a chd_tick
    def chain(base, fanout, joined):
        def setup(chd):
            e = base(chd)
            e.begin_interest(e._rules_batch[0], MS, with_fanout=fanout)
            if joined:
                e.tick(None, MS, chd.capi.TICK_BUILD)
            return e
        return setup

    for base in (followed, rings, comm_rings):
        for fanout in (True, False):
            for joined in (False, True):
                out[base.__name__ + "_chain" + ("_fanout" if fanout else "") + ("_joined" if joined else "")] = chain(base, fanout, joined)
    return out


SETUPS = _setups()


# ---------------------------------------------------------------------------------------------------------------- gated calls
def _calls():
    def p(a):
        from channeld_b200.capi import ptr

        return ptr(a)

    def view_entity_id(chd, e, want_count=None):
        q, n = C.c_void_p(), C.c_uint64()
        st = chd.L.chd_device_view(e.h, chd.capi.VIEW_ENTITY_ID, C.byref(q), C.byref(n))
        if want_count is not None and st == OK:
            assert n.value == want_count
        return st

    def tick_delta(chd, e):
        return _status(lambda: e.tick(e._rules_batch[0], 0, DELTA_FLAGS))

    def tick_build_delta(chd, e):
        return _status(lambda: e.tick(e._rules_batch[0], 0, chd.capi.TICK_BUILD | chd.capi.TICK_VISIBLE_DELTA))

    def tick_sharded(chd, e):
        b, keep = chd.engine.make_batch(0)
        return chd.L.chd_tick_sharded(e.h, C.byref(b), 0, chd.capi.TICK_ALL, None)

    def visible_delta_with_entries(chd, e):
        st = chd.L.chd_visible_delta(e.h)
        if st == OK:
            assert e.visible_delta_counts()[0] > 0
        return st

    def export_border_named_by_table_id(chd, e):
        import torch

        cnt = C.c_uint32()
        d = torch.full((32,), -1, dtype=torch.int32, device="cuda")
        st = chd.L.chd_export_border(e.h, p(d), 16, C.byref(cnt))
        if st == OK:  # both are border records, named by table id
            assert cnt.value == 2
            assert sorted(d[:4].cpu().numpy().view(np.uint32)[::2].tolist()) == [5, 6]
        return st

    def import_halo_then_build(chd, e):
        import torch

        d = torch.full((32,), -1, dtype=torch.int32, device="cuda")
        e.export_border(d, 16)
        st = chd.L.chd_import_halo(e.h, p(d), 2, 0, 2)
        if st == OK:
            e.build()
            assert sorted(e.get_cells()[1].tolist()) == [5, 6]
        return st

    def handoff(chd, e):
        n = C.c_uint32()
        return chd.L.chd_handoff_entities(e.h, None, None, None, None, 0, C.byref(n))

    def export_ring_limits(chd, e):
        import torch

        cnt = C.c_uint32()
        d = torch.zeros(64, dtype=torch.int32, device="cuda")
        return chd.L.chd_export_ring_limits(e.h, p(d), 32, C.byref(cnt))

    def adjacent_broadcast(chd, e):
        off = np.zeros(1, np.uint32)
        return chd.L.chd_adjacent_broadcast(e.h, C.byref(chd.capi.BroadcastBatch(n=0)), None, p(off), None, 0)

    def adopt_queries(chd, e):
        e.prefetch_queries(*e._rules_batch)
        return chd.L.chd_adopt_prefetched(e.h)

    def batch(e):
        return C.byref(e._rules_batch[0])

    calls = {
        # rule 1
        "set_entities": lambda chd, e: chd.L.chd_set_entities(e.h, p(X4), p(Z4), 4),
        "prefetch_entities": lambda chd, e: chd.L.chd_prefetch_entities(e.h, p(X4), p(Z4), 4),
        "set_entities_f32": lambda chd, e: chd.L.chd_set_entities_f32(e.h, p(XF), p(ZF), 4),
        "prefetch_entities_f32": lambda chd, e: chd.L.chd_prefetch_entities_f32(e.h, p(XF), p(ZF), 4),
        "entity_buffers": lambda chd, e: chd.L.chd_entity_buffers(e.h, None, None, None),
        "set_entity_count": lambda chd, e: chd.L.chd_set_entity_count(e.h, 4),
        "set_entity_ids": lambda chd, e: chd.L.chd_set_entity_ids(e.h, p(GID4), 4),
        "set_slab": lambda chd, e: chd.L.chd_set_slab(e.h, 0, 1, 1),
        "set_slab_wider": lambda chd, e: chd.L.chd_set_slab(e.h, 0, 2, 1),
        "comm_init": lambda chd, e: chd.L.chd_comm_init(e.h, (C.c_uint8 * 128)(), 0, 1, 1, 16, 0, 0),
        # rule 2
        "export_border": lambda chd, e: chd.L.chd_export_border(e.h, None, 0, None),
        "export_border_named_by_table_id": export_border_named_by_table_id,
        "import_halo": lambda chd, e: chd.L.chd_import_halo(e.h, None, 0, 0, 0),
        "import_halo_then_build": import_halo_then_build,
        "tick_sharded": tick_sharded,
        "reserve_visible_delta_ids": lambda chd, e: chd.L.chd_reserve_visible_delta_ids(e.h, 64, ID_SPACE),
        # rule 3
        "spawn_entities": lambda chd, e: chd.L.chd_spawn_entities(e.h, None, None, None, 0, None),
        "spawn_entities_f32": lambda chd, e: chd.L.chd_spawn_entities_f32(e.h, None, None, None, 0, None),
        "despawn_entities": lambda chd, e: chd.L.chd_despawn_entities(e.h, None, 0, None),
        "move_entities": lambda chd, e: chd.L.chd_move_entities(e.h, None, None, None, 0),
        "move_entities_f32": lambda chd, e: chd.L.chd_move_entities_f32(e.h, None, None, None, 0),
        "get_entity_stats": lambda chd, e: chd.L.chd_get_entity_stats(e.h, C.byref(chd.capi.EntityStats())),
        "handoff_entities": handoff,
        "view_entity_id": view_entity_id,
        "view_entity_id_of_one": lambda chd, e: view_entity_id(chd, e, want_count=1),
        # rule 4
        "entity_table_init": lambda chd, e: chd.L.chd_entity_table_init(e.h),
        # rules 5 and 6
        "reserve_visible_delta": lambda chd, e: chd.L.chd_reserve_visible_delta(e.h, 64),
        "reserve_visible_delta_1024": lambda chd, e: chd.L.chd_reserve_visible_delta(e.h, 1024),
        "reserve_visible_delta_ids_n": lambda chd, e: chd.L.chd_reserve_visible_delta_ids(e.h, 64, chd.wc.n_entities),
        "reserve_visible_delta_ids_other_space": lambda chd, e: chd.L.chd_reserve_visible_delta_ids(e.h, 64, 2 * ID_SPACE),
        "reserve_visible_delta_ids_zero_space": lambda chd, e: chd.L.chd_reserve_visible_delta_ids(e.h, 64, 0),
        # rule 7
        "visible_delta": lambda chd, e: chd.L.chd_visible_delta(e.h),
        "visible_delta_with_entries": visible_delta_with_entries,
        "tick_delta": tick_delta,
        "tick_build_delta": tick_build_delta,
        # rule 9
        "follow_bind": lambda chd, e: _status(lambda: e.follow_bind([0], [0], sph_r=[50.0])),
        "follow_unbind": lambda chd, e: chd.L.chd_follow_unbind(e.h, p(np.zeros(1, np.uint32)), 1),
        "follow_queries": lambda chd, e: chd.L.chd_follow_queries(e.h, chd.capi.FOLLOW_ALL),
        "follow_queries_with": lambda chd, e: chd.L.chd_follow_queries_with(e.h, chd.capi.FOLLOW_ALL, batch(e)),
        "follow_queries_with_adopted": lambda chd, e: chd.L.chd_follow_queries_with(e.h, chd.capi.FOLLOW_ALL, None),
        "get_follow": lambda chd, e: chd.L.chd_get_follow(e.h, None, None, None, None, None, 0, None, None),
        "adopt_queries": adopt_queries,
        "begin_interest_waiting": lambda chd, e: chd.L.chd_begin_interest(e.h, None, MS, 1),
        "tick_follow": lambda chd, e: chd.L.chd_tick(e.h, None, MS, chd.capi.TICK_ALL | chd.capi.TICK_FOLLOW, None),
        "tick_sharded_follow": lambda chd, e: chd.L.chd_tick_sharded(e.h, None, MS, chd.capi.TICK_ALL | chd.capi.TICK_FOLLOW, None),
        # rule 10
        "apply_subscriptions": lambda chd, e: chd.L.chd_apply_subscriptions(e.h, C.byref(chd.capi.SubBatch(n=0)), MS, None),
        # rule 11
        "spawn_entities_facing": lambda chd, e: chd.L.chd_spawn_entities_facing(e.h, None, None, None, None, None, 0, None),
        "follow_set_frame": lambda chd, e: chd.L.chd_follow_set_frame(e.h, C.byref(chd.capi.FollowFrameBatch(n=0))),
        "get_follow_frame": lambda chd, e: chd.L.chd_get_follow_frame(e.h, None, None, None, None, None, None, None, 0, None),
        # rule 12
        "export_ring_limits": export_ring_limits,
        "import_ring_limits": lambda chd, e: chd.L.chd_import_ring_limits(e.h, None, 0),
        "rings_append": lambda chd, e: chd.L.chd_rings_append(e.h, p(RING_OFF), 0, None, None),
        "get_rings": lambda chd, e: chd.L.chd_get_rings(e.h, p(RING_OFF), None, None, None, None, 0),
        "begin_interest": lambda chd, e: chd.L.chd_begin_interest(e.h, batch(e), MS, 1),
        "update_interest": lambda chd, e: chd.L.chd_update_interest(e.h, batch(e), MS),
        "tick": lambda chd, e: chd.L.chd_tick(e.h, batch(e), MS, chd.capi.TICK_ALL, None),
        "tick_sharded_batch": lambda chd, e: chd.L.chd_tick_sharded(e.h, batch(e), MS, chd.capi.TICK_ALL, None),
        # rule 13
        "set_rings": lambda chd, e: chd.L.chd_set_rings(e.h, p(RING_OFF), 0, None, None, None, None),
        "rings_init": lambda chd, e: chd.L.chd_rings_init(e.h, 513),
        "set_channel_start_times": lambda chd, e: chd.L.chd_set_channel_start_times(e.h, None),
        "adjacent_broadcast": adjacent_broadcast,
    }
    return calls


CALLS = _calls()

RULE1 = ["set_entities", "prefetch_entities", "set_entities_f32", "prefetch_entities_f32", "entity_buffers", "set_entity_count", "set_entity_ids",
         "set_slab", "comm_init"]
RULE2 = ["export_border", "import_halo", "tick_sharded", "reserve_visible_delta_ids"]
CHAIN = ["begin_interest", "rings_init", "set_channel_start_times", "follow_queries", "follow_queries_with", "get_follow", "get_follow_frame",
         "apply_subscriptions", "adjacent_broadcast"]
CHAIN_COMM = ["export_ring_limits", "import_ring_limits", "tick_sharded_batch"]
RULE3 = ["spawn_entities", "spawn_entities_f32", "despawn_entities", "move_entities", "move_entities_f32", "get_entity_stats", "handoff_entities",
         "view_entity_id"]

# rule -> its rows (set-up, gated call, status)
RULES = {
    # 1. table mode refuses the calls that bypass the table, slab or not
    1: [("table", c, STATE) for c in RULE1] + [("table_slab", c, STATE) for c in ("set_slab_wider", "comm_init", "set_entities", "set_entity_ids")],
    # 2. the multi-GPU calls need a table engine made a slab first
    2: [("table", c, STATE) for c in RULE2] + [("table_slab", "reserve_visible_delta_ids", OK),
                                                ("table_slab_spawned", "export_border_named_by_table_id", OK),
                                                ("table_slab_spawned", "import_halo_then_build", OK)],
    # 3. the calls by id need table mode
    3: [("fresh", c, STATE) for c in RULE3] + [("table_built", "view_entity_id_of_one", OK)],
    # 4. chd_entity_table_init needs a fresh engine (a slab may come first)
    4: [(s, "entity_table_init", STATE) for s in ("table", "built", "assigned_without_ids", "ids_null", "id_delta", "slab_ids", "slab_assigned",
                                                  "slab_built", "slab_delta_ids")]
    + [(s, "entity_table_init", OK) for s in ("fresh", "slab", "slab_ids_null")],
    # 5. index-mode deltas are single-GPU only: refused after a slab or global ids, unless id mode is on
    5: [(s, c, STATE) for s in ("index_delta_then_slab", "index_delta_then_ids") for c in ("reserve_visible_delta_1024", "visible_delta", "tick_build_delta")]
    + [("table_slab", "reserve_visible_delta", STATE), ("slab", "reserve_visible_delta", STATE), ("id_delta", "reserve_visible_delta", OK)],
    # 6. chd_reserve_visible_delta_ids: one id_space, never after index mode
    6: [("fresh", "reserve_visible_delta_ids_zero_space", INVALID), ("id_delta", "reserve_visible_delta_ids_other_space", INVALID),
        ("id_delta", "reserve_visible_delta_ids", OK), ("index_delta", "reserve_visible_delta_ids_n", STATE)],
    # 7. a delta runs after a reserve, in id mode only with ids, and on a build of the current state
    7: [("fresh", "visible_delta", STATE), ("id_delta_without_ids", "tick_delta", STATE), ("id_delta_without_ids_built", "visible_delta", STATE),
        ("id_delta_ids_after_build", "visible_delta", STATE), ("id_delta_ids_built", "visible_delta_with_entries", OK),
        ("table_spawned_after_build", "visible_delta", STATE), ("table_built", "visible_delta", OK)],
    # 8. the halo import needs a cell assignment and global ids
    8: [("fresh", "import_halo", STATE), ("assigned_without_ids", "import_halo", STATE)],
    # 9. no followers on an index-mode slab, no slab once a slot follows; one query batch per interest update, and an update that
    # takes the waiting batch needs one
    9: [("slab_subscribed", c, STATE) for c in ("follow_bind", "follow_unbind", "follow_queries", "follow_queries_with", "get_follow")]
    + [("following_index", c, STATE) for c in ("set_slab", "comm_init")]
    + [("generated", c, STATE) for c in ("follow_queries", "follow_queries_with", "adopt_queries", "get_follow", "get_follow_frame")]
    + [("generated", c, OK) for c in ("tick_follow", "begin_interest_waiting")]
    + [("adopted", c, STATE) for c in ("follow_queries", "follow_queries_with", "tick_follow")]
    + [("adopted", c, OK) for c in ("follow_queries_with_adopted", "begin_interest_waiting")]
    + [("followed", c, STATE) for c in ("begin_interest_waiting", "tick_follow", "follow_queries_with_adopted")]
    + [("followed", c, OK) for c in ("follow_queries", "get_follow", "get_follow_frame", "adopt_queries")]
    + [("comm_rings", "tick_sharded_follow", STATE)],
    # 10. explicit subscriptions are refused on a slab
    10: [("slab", "apply_subscriptions", STATE), ("fresh", "apply_subscriptions", OK)],
    # 11. facings and frames need entity-table mode
    11: [("fresh", c, STATE) for c in ("spawn_entities_facing", "follow_set_frame", "get_follow_frame")]
    + [("table", "spawn_entities_facing", OK), ("followed", "follow_set_frame", OK), ("followed", "get_follow_frame", OK)],
    # 12. ring limits need device rings on a slab; a communicator engine's staged updates hold off what would read or raise around them
    12: [(s, c, STATE) for s in ("slab", "rings") for c in ("export_ring_limits", "import_ring_limits")]
    + [("comm_rings", c, OK) for c in ("export_ring_limits", "import_ring_limits")]
    + [("comm_rings_staged", c, STATE) for c in ("rings_append", "get_rings", "begin_interest", "update_interest", "tick")]
    + [("comm_rings_staged", "tick_sharded_batch", OK)],
    # 13. a begun chd_begin_interest refuses what its chain reads or writes until the chd_tick that joins it: chd_set_rings only when
    # the chain includes the fan-out, chd_tick_sharded only with device rings
    13: [("followed_chain" + v, c, STATE) for v in ("_fanout", "") for c in CHAIN]
    + [("followed_chain_fanout", "set_rings", STATE), ("followed_chain", "set_rings", OK)]
    + [("rings_chain" + v, "rings_append", STATE) for v in ("_fanout", "")]
    + [("comm_rings_chain" + v, c, STATE) for v in ("_fanout", "") for c in CHAIN_COMM]
    + [("followed_chain" + v + "_joined", c, OK) for v in ("_fanout", "") for c in CHAIN + ["set_rings"]]
    + [("rings_chain" + v + "_joined", "rings_append", OK) for v in ("_fanout", "")]
    + [("comm_rings_chain" + v + "_joined", c, OK) for v in ("_fanout", "") for c in CHAIN_COMM],
}


def _check(chd, rule, refusal=None):
    """runs every row of the rule on a fresh engine and reports all the rows that break it at once; `refusal`: text every refusal's
    error contains"""
    bad = []
    for setup, call, want in RULES[rule]:
        e = SETUPS[setup](chd)
        try:
            got = CALLS[call](chd, e)
            err = chd.L.chd_last_error(e.h).decode()
            if got != want:
                bad.append("%s / %s: status %d, want %d (%s)" % (setup, call, got, want, err))
            elif refusal and got == STATE and refusal not in err:
                bad.append("%s / %s: refused with %r" % (setup, call, err))
        except AssertionError as ex:
            bad.append("%s / %s: %s" % (setup, call, ex))
        finally:
            e.close()
    assert not bad, "rule %d:\n" % rule + "\n".join(bad)


def test_rule_1_table_mode_refuses_the_calls_that_bypass_the_table(chd):
    _check(chd, 1)


def test_rule_2_multi_gpu_calls_need_a_table_engine_made_a_slab_first(chd):
    _check(chd, 2)


def test_rule_3_calls_by_id_need_table_mode(chd):
    _check(chd, 3)


def test_rule_4_table_init_needs_a_fresh_engine(chd):
    _check(chd, 4)


def test_rule_5_index_mode_deltas_are_single_gpu_only(chd):
    _check(chd, 5)


def test_rule_6_id_mode_reserve(chd):
    _check(chd, 6)


def test_rule_7_a_delta_needs_a_reserve_ids_and_a_current_build(chd):
    _check(chd, 7)


def test_rule_8_halo_import_needs_an_assignment_and_global_ids(chd):
    _check(chd, 8)


def test_rule_9_followers_and_one_query_batch_per_interest_update(chd):
    _check(chd, 9)


def test_rule_10_explicit_subscriptions_are_refused_on_a_slab(chd):
    _check(chd, 10)


def test_rule_11_facings_and_frames_need_table_mode(chd):
    _check(chd, 11)


def test_rule_12_ring_limits_need_device_rings_on_a_slab(chd):
    _check(chd, 12)


def test_rule_13_a_begun_interest_chain_holds_off_its_inputs_until_the_tick_joins_it(chd):
    _check(chd, 13, refusal="chd_begin_interest is pending")
