"""Entity-table mode on X-slabs: each rank's table holds the entities it owns, border records and halo imports carry table ids, and
chd_handoff_entities moves an entity to the rank that owns its column by id, with its exact position.  Slab engines on one device
are fed through sharding.EntityRouter and checked every tick against one whole-world table engine fed the same event stream.
Run on an H100:  python -m pytest tests/test_gpu_sharded_table.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_sharded_delta import EMPTY, _batch, _check_delta, _keys

pytestmark = pytest.mark.gpu

MS = 1_000_000
VIS_FLAGS = 1 | 2  # TICK_BUILD | TICK_EMIT
DELTA_FLAGS = 1 | 2 | 16  # ... | TICK_VISIBLE_DELTA
ID_SPACE = 1 << 20


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine, sharding, synth

    capi.lib()

    class NS:
        pass

    ns = NS()
    ns.capi, ns.engine, ns.sharding, ns.synth = capi, engine, sharding, synth
    return ns


def _u32_view(e, which):
    """A u32 device view (chd_device_view) copied to the host."""
    import torch

    e.sync()
    p, n = e.device_view(which)
    if not n:
        return np.zeros(0, np.uint32)

    class _Dev:
        __cuda_array_interface__ = {"shape": (int(n),), "typestr": "<i4", "data": (int(p), False), "version": 3}

    return torch.as_tensor(_Dev(), device="cuda").cpu().numpy().view(np.uint32)


def _live_ids(chd, e):
    ids = _u32_view(e, chd.capi.VIEW_ENTITY_ID)
    return set(ids[ids != 0].tolist())


def _handover_set(e, n):
    a, b, c = e.get_handover(n)
    return set(zip(a.tolist(), b.tolist(), c.tolist()))


def _vis_sets(off, ent):
    return [set(ent[off[j]:off[j + 1]].tolist()) for j in range(len(off) - 1)]


class Events:
    """A seeded table event stream over a world: random ids spawned at random places (a few outside the world), moves (small steps,
    jumps anywhere in the world that cross slab borders, trips out of the world and back), despawns, fresh spawns."""

    def __init__(self, wc, seed):
        self.wc, self.rng = wc, np.random.default_rng(seed)
        self.lo, self.hi = wc.offx, wc.offx + wc.w * wc.cols
        self.zlo, self.zhi = wc.offz, wc.offz + wc.h * wc.rows
        self.pos, self.out, self.used = {}, set(), set()

    def _ids(self, k):
        out = []
        while len(out) < k:
            i = int(self.rng.integers(1, ID_SPACE))
            if i not in self.used:
                self.used.add(i)
                out.append(i)
        return np.array(out, np.uint32)

    def _places(self, k):
        return self.rng.uniform(self.lo, self.hi, k), self.rng.uniform(self.zlo, self.zhi, k)

    def spawn(self, k, n_out=0):
        ids = self._ids(k)
        x, z = self._places(k)
        x[:n_out] = self.lo - 3000.0
        for j, i in enumerate(ids.tolist()):
            self.pos[i] = (x[j], z[j])
            if j < n_out:
                self.out.add(i)
        return ids, x, z

    def tick(self, frozen=()):
        """-> (spawn, move, despawn); ids in `frozen` are not moved."""
        live = np.array(sorted(set(self.pos) - set(frozen)), np.int64)
        pick = self.rng.permutation(live)
        n = len(pick)
        step, jump, leave, gone = np.split(pick, np.cumsum([n // 3, n // 25, n // 100, n // 100]))[:4]
        mids, mx, mz = [], [], []
        for i in step.tolist():
            x, z = self.pos[i]
            if i in self.out:  # back into the world
                x, z = self._places(1)
                x, z = x[0], z[0]
                self.out.discard(i)
            else:
                x = float(np.clip(x + self.rng.uniform(-900, 900), self.lo, self.hi - 1e-6))
                z = float(np.clip(z + self.rng.uniform(-900, 900), self.zlo, self.zhi - 1e-6))
            mids.append(i), mx.append(x), mz.append(z)
        for i in jump.tolist():
            x, z = self._places(1)
            self.out.discard(i)
            mids.append(i), mx.append(x[0]), mz.append(z[0])
        for i in leave.tolist():
            self.out.add(i)
            mids.append(i), mx.append(self.hi + 3000.0), mz.append(self.pos[i][1])
        for i, x, z in zip(mids, mx, mz):
            self.pos[i] = (x, z)
        for i in gone.tolist():
            del self.pos[i]
            self.out.discard(i)
        sp = self.spawn(max(n // 100, 4), n_out=1)
        return sp, (np.array(mids, np.uint32), np.array(mx), np.array(mz)), gone.astype(np.uint32)


NO_MOVES = (np.zeros(0, np.uint32), np.zeros(0), np.zeros(0))


def _apply(e, sp, mv, dp):
    if len(sp[0]):
        assert (e.spawn_entities(*sp) == 0).all()
    if len(mv[0]):
        e.move_entities(*mv)
    if len(dp):
        assert (e.despawn_entities(dp) == 0).all()


def _summary(chd, e):
    s = chd.capi.TickSummary()
    assert chd.capi.lib().chd_summary(e.h, C.byref(s)) == chd.capi.OK and s.overflow == 0
    return s


def _column_owner(chd, ch, wc, world):
    cell = np.asarray(ch, np.int64) - chd.engine.SPATIAL_CHANNEL_ID_START
    return chd.sharding.owner_of_column(cell % wc.cols, wc.cols, world)


# ------------------------------------------------------------------------------------------------- 1. slabs, building blocks
@pytest.mark.parametrize("world", [2, 3])
def test_table_mode_on_slabs_through_the_building_blocks(chd, world):
    """World-many table-mode slab engines on one device (border export, concatenation, halo import, build, interest update, id-mode
    delta, emit) and a whole-world table engine take the same events; the router sends each to its owner and turns hand-off lists
    into adoptions.  Every tick: per connection the visible set equals the whole world's, the ranks' handover lists together are the
    whole world's (each change once), after the hand-offs every live id lives on exactly one rank, and each rank's delta is the set
    difference of its visible lists.  An adopted entity stands still for one tick: its new owner reports a cell change before its
    next cell assignment as part of the spawn (chd_gpu.h)."""
    import torch

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 20_000, 1_000)
    S = wc.n_subscribers
    radius = 1000.0
    halo = chd.sharding.halo_columns(radius, wc.w)
    ev = Events(wc, 100 + world)
    router = chd.sharding.EntityRouter(world, wc.cols, wc.offx, wc.w)
    first = ev.spawn(wc.n_entities, n_out=20)
    own_cap, cap = 2 * wc.n_entities, wc.n_entities
    # subscribers stand still, each on the rank that owns its column
    cx, cz = first[1][20: 20 + S * 10: 10].copy(), first[2][20: 20 + S * 10: 10].copy()  # (the first 20 are outside the world)
    sub_owner = router.owner_of_x(cx)
    subs = [np.nonzero(sub_owner == r_)[0] for r_ in range(world)]
    whole = chd.engine.Engine(wc.cfg(), own_cap, S, max_visible=1 << 25)
    whole.entity_table_init()
    whole.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    engines = []
    for r_ in range(world):
        e = chd.engine.Engine(wc.cfg(), own_cap + cap * world + 16, len(subs[r_]), max_visible=1 << 25)
        e.set_slab(*chd.sharding.slab_columns(wc.cols, world, r_), halo)  # the slab first, then the table
        e.entity_table_init()
        e.set_subscribers(np.asarray(subs[r_] + 1, np.uint32))
        e.reserve_visible_delta_ids(1 << 22, ID_SPACE)
        engines.append(e)
    recs = [torch.empty(2 * cap, dtype=torch.int32, device="cuda") for _ in range(world)]
    prev = [EMPTY] * world
    prev_own = [set() for _ in range(world)]
    frozen = set()
    handed = crossing = transitions = changes = 0
    for t in range(7):
        sp, mv, dp = (first, NO_MOVES, np.zeros(0, np.uint32)) if t == 0 else ev.tick(frozen)
        _apply(whole, sp, mv, dp)
        for r_, (a, b, c) in enumerate(zip(router.spawn(*sp), router.move(*mv), router.despawn(dp))):
            _apply(engines[r_], a, b, c)
        own_now = [set(i for i, o in router.owner.items() if o == r_) for r_ in range(world)]
        batch, keep = _batch(chd, np.arange(S), cx, cz, np.full(S, radius))
        sw = whole.tick(batch, t * 33 * MS, VIS_FLAGS)
        assert sw.overflow == 0
        w_vis = _vis_sets(*whole.get_visible())
        w_ho = _handover_set(whole, sw.n_handover)
        for r_, e in enumerate(engines):
            assert e.export_border(recs[r_], cap) <= cap
        torch.cuda.synchronize()
        gathered = torch.cat(recs)
        torch.cuda.synchronize()
        ho_union, ho_total = set(), 0
        for r_, e in enumerate(engines):
            e.import_halo(gathered, cap * world, r_ * cap, cap)
            e.build()
            n = len(subs[r_])
            batch, keep = _batch(chd, np.arange(n), cx[subs[r_]], cz[subs[r_]], np.full(n, radius))
            e.update_interest(batch, t * 33 * MS)
            e.visible_delta()
            e.emit_visible()
            s = _summary(chd, e)
            now = e.get_visible()
            for k, v in enumerate(_vis_sets(*now)):
                assert v == w_vis[subs[r_][k]], (t, r_, k)
            ho = _handover_set(e, s.n_handover)
            ho_union |= ho
            ho_total += len(ho)
            d = e.get_visible_delta()
            _check_delta(d, prev[r_], now)
            if t:
                changes += len(d[1]) + len(d[3])
                kept = np.intersect1d(_keys(*prev[r_], n), _keys(*now, n))
                kept_ids = (kept & np.uint64(0xFFFFFFFF)).astype(np.int64)
                became_own = np.fromiter(own_now[r_] - prev_own[r_], np.int64)
                transitions += int(np.isin(kept_ids, became_own).sum())
            prev[r_], prev_own[r_] = now, own_now[r_]
        del gathered
        assert ho_union == w_ho and ho_total == len(w_ho), t
        inside = [(src, dst) for _, src, dst in w_ho if src and dst]
        if inside:
            a, b = zip(*inside)
            crossing += int((_column_owner(chd, a, wc, world) != _column_owner(chd, b, wc, world)).sum())
        # hand-offs after the tick.  Engines without a communicator do not know the rank count (dst_rank is computed for a world of
        # one), so the router's own column owner names the destination here; it is never the giver.
        lists = []
        for r_, e in enumerate(engines):
            ids, dst, x, z = e.handoff_entities()
            owner = chd.sharding.owner_of_column(chd.sharding.column_of(x, wc.offx, wc.w, wc.cols), wc.cols, world)
            assert not (owner == r_).any() and (chd.sharding.column_of(x, wc.offx, wc.w, wc.cols) >= 0).all()
            lists.append((ids, owner, x, z))
            handed += len(ids)
        adopt = router.handoff(lists)
        frozen = set()
        for r_, (ids, x, z) in enumerate(adopt):
            if len(ids):
                assert (engines[r_].spawn_entities(ids, x, z) == 0).all()
                frozen |= set(ids.tolist())
        live = [_live_ids(chd, e) for e in engines]
        assert sum(len(v) for v in live) == len(set().union(*live)) == len(_live_ids(chd, whole))
        assert set().union(*live) == _live_ids(chd, whole) == set(router.owner)
        for r_ in range(world):
            assert live[r_] == set(i for i, o in router.owner.items() if o == r_)
        assert sum(e.entity_stats()["live"] for e in engines) == whole.entity_stats()["live"]
    assert handed > 0 and crossing > 0 and transitions > 0 and changes > 0, (handed, crossing, transitions, changes)
    for e in engines + [whole]:
        e.close()


# ---------------------------------------------------------------------------------------------- 2. hand-off exactness and rules
def test_handoff_is_exact_transactional_and_refused_where_it_must_be(chd):
    import torch

    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 4_000, 16)
    L, capi = chd.capi.lib(), chd.capi
    lo, hi = chd.sharding.slab_columns(wc.cols, 2, 0)
    xmid = wc.offx + hi * wc.w  # first x of rank 1's slab
    cap = 4_096
    recs = torch.empty(2 * cap, dtype=torch.int32, device="cuda")

    def status(call):
        with pytest.raises(capi.ChdError) as ei:
            call()
        return ei.value.status

    def engine(rank):
        e = chd.engine.Engine(wc.cfg(), 3 * cap, 16)
        e.set_slab(*chd.sharding.slab_columns(wc.cols, 2, rank), 1)
        e.entity_table_init()
        return e

    a, b = engine(0), engine(1)
    n = C.c_uint32()
    assert L.chd_handoff_entities(a.h, None, None, None, None, 0, C.byref(n)) == capi.ERR_STATE  # before any cell assignment
    rng = np.random.default_rng(5)
    ids = np.arange(1, 201, dtype=np.uint32)
    x = rng.uniform(wc.offx, xmid - 1.0, 200)
    z = rng.uniform(wc.offz, wc.offz + wc.h * wc.rows, 200)
    assert (a.spawn_entities(ids[:100], x[:100], z[:100]) == 0).all()
    assert (a.spawn_entities_f32(ids[100:], x[100:].astype(np.float32), z[100:].astype(np.float32)) == 0).all()
    a.export_border(recs, cap)
    assert a.handoff_entities()[0].size == 0  # nobody outside the slab yet
    # into rank 1's slab: f64 positions that no float holds, f32 positions, and one that stays
    xs = np.nextafter(rng.uniform(xmid + 10.0, wc.offx + wc.w * wc.cols - 10.0, 40), np.inf)
    zs = np.nextafter(z[:40] + 0.1, -np.inf)
    a.move_entities(ids[:20], xs[:20], zs[:20])
    a.move_entities_f32(ids[20:40], xs[20:40].astype(np.float32), zs[20:40].astype(np.float32))
    a.move_entities(ids[40:41], [wc.offx + 1.0], [wc.offz + 1.0])
    late = np.arange(301, 306, dtype=np.uint32)  # spawned (f32) straight into the other slab
    assert (a.spawn_entities_f32(late, xs[:5].astype(np.float32) + 1, zs[:5].astype(np.float32)) == 0).all()
    moved = np.concatenate([ids[:40], late])
    want_x = np.concatenate([xs[:20], xs[20:40].astype(np.float32).astype(np.float64), (xs[:5].astype(np.float32) + 1).astype(np.float64)])
    want_z = np.concatenate([zs[:20], zs[20:40].astype(np.float32).astype(np.float64), zs[:5].astype(np.float32).astype(np.float64)])
    assert L.chd_handoff_entities(a.h, None, None, None, None, 0, C.byref(n)) == capi.ERR_STATE  # events since the assignment
    a.export_border(recs, cap)
    slots_before = _u32_view(a, capi.VIEW_ENTITY_ID)
    # too small a buffer: CHD_ERR_CAPACITY, the count, nothing removed
    small = [np.zeros(8, np.uint32), np.zeros(8, np.uint32), np.zeros(8), np.zeros(8)]
    assert L.chd_handoff_entities(a.h, *[capi.ptr(v) for v in small], 8, C.byref(n)) == capi.ERR_CAPACITY and n.value == 45
    assert a.entity_stats()["live"] == 205
    np.testing.assert_array_equal(_u32_view(a, capi.VIEW_ENTITY_ID), slots_before)
    rid, rdst, rn = a.get_rehome()  # read-only, names ids
    assert rn == 45 and set(rid.tolist()) == set(moved.tolist())
    got_id, got_dst, got_x, got_z = a.handoff_entities(cap=8)  # grows the buffer and asks again: the same set
    order = np.argsort(got_id)
    np.testing.assert_array_equal(got_id[order], moved)
    np.testing.assert_array_equal(got_x[order].view(np.uint64), want_x.view(np.uint64))  # bit-exact, f32 widened included
    np.testing.assert_array_equal(got_z[order].view(np.uint64), want_z.view(np.uint64))
    np.testing.assert_array_equal(np.sort(got_dst), np.sort(rdst))
    st = a.entity_stats()
    assert st["live"] == 160 and st["quarantined"] == 0 and st["high_water"] == 205
    assert status(a.handoff_entities) == capi.ERR_STATE  # the hand-off itself is an event
    # the giver's slots are free at once and reused first in, first out (in the order the list gave them up)
    freed = np.nonzero(np.isin(slots_before, got_id))[0]
    assert (_u32_view(a, capi.VIEW_ENTITY_ID)[freed] == 0).all()
    fresh = np.arange(1000, 1045, dtype=np.uint32)
    assert (a.spawn_entities(fresh, np.full(45, wc.offx + 5.0), np.full(45, wc.offz + 5.0)) == 0).all()
    np.testing.assert_array_equal(_u32_view(a, capi.VIEW_ENTITY_ID)[np.sort(freed)], fresh)
    # adoption is a spawn on the receiver: the entities sit in its cell CSR under their ids, in the cells of their positions
    assert (b.spawn_entities(got_id, got_x, got_z) == 0).all()
    b.export_border(recs, cap)
    b.import_halo(recs, 0, 0, 0)
    b.build()
    cs, se = b.get_cells()
    cell_of = np.repeat(np.arange(len(cs) - 1), np.diff(cs.astype(np.int64)))
    where = dict(zip(se.tolist(), cell_of.tolist()))
    want_cell = b.cell_of(got_x, got_z)
    for i, c in zip(got_id.tolist(), (want_cell - chd.engine.SPATIAL_CHANNEL_ID_START).tolist()):
        assert where[i] == c
    # refusals: outside table mode; index-mode deltas, entity ids and a new slab on a table slab engine; the slab calls on a table
    # engine that was not made a slab before chd_entity_table_init
    plain = chd.engine.Engine(wc.cfg(), 64, 4)
    assert L.chd_handoff_entities(plain.h, None, None, None, None, 0, C.byref(n)) == capi.ERR_STATE
    assert status(lambda: a.reserve_visible_delta(64)) == capi.ERR_STATE
    assert status(lambda: a.set_entity_ids(np.arange(4, dtype=np.uint32))) == capi.ERR_STATE
    assert status(lambda: a.set_slab(0, 2, 1)) == capi.ERR_STATE
    single = chd.engine.Engine(wc.cfg(), 64, 4)
    single.entity_table_init()
    assert L.chd_export_border(single.h, capi.ptr(recs), cap, None) == capi.ERR_STATE
    assert status(lambda: single.reserve_visible_delta_ids(64, 1 << 10)) == capi.ERR_STATE
    ids_first = chd.engine.Engine(wc.cfg(), 64, 4)
    ids_first.set_slab(0, 2, 1)
    ids_first.set_entity_ids(np.arange(4, dtype=np.uint32))
    assert status(ids_first.entity_table_init) == capi.ERR_STATE
    assert L.chd_handoff_entities(None, None, None, None, None, 0, C.byref(n)) == capi.ERR_INVALID
    for e in (a, b, plain, single, ids_first):
        e.close()


def test_id_mode_respawn_of_one_id_between_deltas_is_not_reported(chd):
    """Id mode names ids: a despawn followed by a spawn of the same id (here into another slot) between two deltas gives no entries
    where a slot sees the id in both states, and no slot is quarantined (the freed slot goes to the next spawn)."""
    wc = chd.synth.scaled(chd.synth.CONFIGS["2x2"], 64, 1)
    e = chd.engine.Engine(wc.cfg(), 64, 1)
    e.set_slab(0, wc.cols, 1)  # a one-slab world: id-mode deltas in table mode are the slab engines' mode
    e.entity_table_init()
    e.set_subscribers(np.array([1], np.uint32))
    e.reserve_visible_delta_ids(1 << 10, 1 << 10)
    batch, keep = _batch(chd, [0], [-1000.0], [-1000.0], [300.0])
    assert (e.spawn_entities([7, 8], [-1000.0, -1100.0], [-1000.0, -1000.0]) == 0).all()
    e.tick(batch, 0, DELTA_FLAGS)
    eo, en, lo, le = e.get_visible_delta()
    assert sorted(en.tolist()) == [7, 8] and len(le) == 0
    assert (e.despawn_entities([7]) == 0).all()
    assert (e.spawn_entities([9], [-1050.0], [-1000.0]) == 0).all()  # takes 7's slot at once: no quarantine
    assert (e.spawn_entities([7], [-1010.0], [-1000.0]) == 0).all()  # 7 again, in a fresh slot
    assert e.entity_stats()["quarantined"] == 0 and e.entity_stats()["high_water"] == 3
    e.tick(batch, 33 * MS, DELTA_FLAGS)
    eo, en, lo, le = e.get_visible_delta()
    assert en.tolist() == [9] and len(le) == 0
    e.close()


# ---------------------------------------------------------------------------------------- 3. chd_tick_sharded at world one
@pytest.mark.parametrize("graphs", [True, False])
def test_tick_sharded_table_mode_at_world_one_matches_a_single_engine(chd, graphs):
    """chd_tick_sharded on a one-rank communicator in table mode gives the arrays that a table engine over the whole grid, driven by
    chd_tick without any exchange, gives for the same events: sorted ids, visible lists and id-mode deltas element for element, the same handover list (compared sorted: it is filled
    by atomic appends), and no hand-offs."""
    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 20_000, 1_000)
    S = wc.n_subscribers
    radius = 1000.0
    cap = wc.n_entities
    ev = Events(wc, 7)
    first = ev.spawn(wc.n_entities, n_out=20)
    cx, cz = first[1][20: 20 + S * 10: 10].copy(), first[2][20: 20 + S * 10: 10].copy()
    sh = chd.engine.Engine(wc.cfg(), 2 * wc.n_entities + cap + 16, S, max_visible=1 << 25)
    one = chd.engine.Engine(wc.cfg(), 2 * wc.n_entities, S, max_visible=1 << 25)
    sh.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, chd.sharding.halo_columns(radius, wc.w), cap)
    sh.entity_table_init()
    one.set_slab(0, wc.cols, 1)  # (the whole grid: id-mode deltas in table mode need a slab engine)
    one.entity_table_init()
    for e in (sh, one):
        e.enable_graphs(graphs)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.reserve_visible_delta_ids(1 << 22, ID_SPACE)
    n_ho = 0
    for t in range(7):
        sp, mv, dp = (first, NO_MOVES, np.zeros(0, np.uint32)) if t == 0 else ev.tick()
        batch, keep = _batch(chd, np.arange(S), cx, cz, np.full(S, radius))
        for e in (sh, one):
            _apply(e, sp, mv, dp)
        s1 = sh.tick_sharded(batch, t * 33 * MS, DELTA_FLAGS)
        s2 = one.tick(batch, t * 33 * MS, DELTA_FLAGS)
        assert s1.overflow == 0 and s2.overflow == 0 and s1.n_handover == s2.n_handover
        for u, v in zip(sh.get_cells(), one.get_cells()):
            np.testing.assert_array_equal(u, v)
        for u, v in zip(sh.get_visible(), one.get_visible()):
            np.testing.assert_array_equal(u, v)
        assert sorted(_handover_set(sh, s1.n_handover)) == sorted(_handover_set(one, s2.n_handover))
        n_ho += s1.n_handover
        for u, v in zip(sh.get_visible_delta(), one.get_visible_delta()):
            np.testing.assert_array_equal(u, v)
        assert sh.handoff_entities()[0].size == 0
    assert n_ho > 0
    if graphs:
        assert sh.graph_launch_count() > 0
    assert chd.capi.lib().chd_comm_destroy(sh.h) == chd.capi.OK
    for e in (sh, one):
        e.close()
