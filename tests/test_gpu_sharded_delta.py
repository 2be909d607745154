"""Id-mode visible-set deltas (chd_reserve_visible_delta_ids): entered / left entities per subscriber slot named by GLOBAL id, on a
single engine whose host permutes its entity array every tick, on X-slabs driven through the building blocks (border export, halo
import, build, interest update, delta) with entities re-homed between ticks, and in chd_tick_sharded with subscriber migration.
Every check is against set differences of the same engine's visible lists (global ids) across consecutive deltas.
Run on an H100:  python -m pytest tests/test_gpu_sharded_delta.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MS = 1_000_000
DELTA_FLAGS = 1 | 2 | 16  # TICK_BUILD | TICK_EMIT | TICK_VISIBLE_DELTA


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


def _keys(off, ent, n):
    """CSR by slot -> sorted u64 keys slot << 32 | entity (a per-slot set)"""
    off = np.asarray(off, np.uint64)
    if len(off) < n + 1:
        off = np.concatenate([off, np.full(n + 1 - len(off), off[-1] if len(off) else 0, np.uint64)])
    slot = np.repeat(np.arange(n, dtype=np.uint64), np.diff(off[: n + 1]).astype(np.int64))
    return np.sort((slot << np.uint64(32)) | np.asarray(ent[: len(slot)], np.uint64))


def _check_delta(d, prev_vis, now_vis):
    """d = (enter_off, enter, leave_off, leave) must be, per slot, now \\ prev and prev \\ now (as sets)"""
    eo, en, lo, le = d
    n = max(len(eo), len(prev_vis[0]), len(now_vis[0])) - 1
    pk, nk = _keys(*prev_vis, n), _keys(*now_vis, n)
    np.testing.assert_array_equal(_keys(eo, en, n), nk[~np.isin(nk, pk)])
    np.testing.assert_array_equal(_keys(lo, le, n), pk[~np.isin(pk, nk)])
    # no slot repeats an id inside one list
    for off, ent in ((eo, en), (lo, le)):
        k = _keys(off, ent, n)
        assert len(np.unique(k)) == len(k)


EMPTY = (np.zeros(1, np.uint64), np.zeros(0, np.uint32))


def _world(chd, n_ent, n_sub, name="benchmark"):
    wc = chd.synth.scaled(chd.synth.CONFIGS[name], n_ent, n_sub)
    x, z = chd.synth.entities(wc)
    idx = (np.arange(n_sub, dtype=np.int64) * max(n_ent // n_sub, 1)) % n_ent  # subscriber j stands on entity idx[j]
    return wc, x, z, idx


def _batch(chd, slots, cx, cz, r):
    return chd.engine.make_batch(len(slots), sub=np.asarray(slots, np.uint32), sphere=(np.asarray(cx, np.float64).copy(),
                                                                                       np.asarray(cz, np.float64).copy(),
                                                                                       np.asarray(r, np.float64)))


# ---------------------------------------------------------------------------------------------------------------- 1. one engine
def _permuted_run(chd, graphs):
    wc, x, z, idx = _world(chd, 30_000, 3_000)
    N, S = wc.n_entities, wc.n_subscribers
    r = np.full(S, wc.radius)
    rng = np.random.default_rng(7)
    a = chd.engine.Engine(wc.cfg(), N, S)  # id mode, entity array shuffled every tick
    b = chd.engine.Engine(wc.cfg(), N, S)  # index mode over the unshuffled array
    for e in (a, b):
        e.enable_graphs(graphs)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    a.reserve_visible_delta_ids(1 << 22, N)
    b.reserve_visible_delta(1 << 22)
    prev = EMPTY
    out = []
    changes = 0
    for t in range(8):
        if t:
            x, z = chd.synth.move_entities(wc, x, z, t, 150.0)
        perm = rng.permutation(N)
        a.set_entities(x[perm], z[perm])
        a.set_entity_ids(perm.astype(np.uint32))  # position i is entity perm[i]
        b.set_entities(x, z)
        for e in (a, b):
            batch, keep = _batch(chd, np.arange(S), x[idx], z[idx], r)
            s = e.tick(batch, t * 33 * MS, DELTA_FLAGS)
            assert s.overflow == 0
        now = a.get_visible()
        da, db = a.get_visible_delta(), b.get_visible_delta()
        _check_delta(da, prev, now)
        # the same sets as index mode (whose indices are the global ids here)
        np.testing.assert_array_equal(_keys(da[0], da[1], S), _keys(db[0], db[1], S))
        np.testing.assert_array_equal(_keys(da[2], da[3], S), _keys(db[2], db[3], S))
        if t:
            changes += len(da[1]) + len(da[3])
        out.append(da)
        prev = now
    assert changes > 0
    return out, a.graph_launch_count()


def test_id_mode_on_one_engine_with_a_permuted_entity_array(chd):
    """Per slot, the id-mode delta is the set difference of consecutive get_visible() lists and equals an index-mode engine's
    delta over the unshuffled inputs; with and without CUDA graphs the arrays are identical."""
    on, g_on = _permuted_run(chd, True)
    off, g_off = _permuted_run(chd, False)
    assert g_on > 0 and g_off == 0
    for u, v in zip(on, off):
        for p, q in zip(u, v):
            np.testing.assert_array_equal(p, q)


def test_id_mode_launches_one_kernel_more_than_index_mode(chd):
    """The id-mode stage is the index-mode stage plus the key scatter (its memsets are not kernels); index mode is unchanged."""
    wc, x, z, idx = _world(chd, 20_000, 2_000)
    N, S = wc.n_entities, wc.n_subscribers
    counts = []
    for ids in (False, True):
        e = chd.engine.Engine(wc.cfg(), N, S)
        e.enable_graphs(False)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        if ids:
            e.reserve_visible_delta_ids(1 << 20, N)
            e.set_entity_ids(np.arange(N, dtype=np.uint32))
        else:
            e.reserve_visible_delta(1 << 20)
        e.set_entities(x, z)
        batch, keep = _batch(chd, np.arange(S), x[idx], z[idx], np.full(S, wc.radius))
        e.tick(batch, 0, DELTA_FLAGS)
        n0 = e.launch_count()
        e.visible_delta()
        counts.append(e.launch_count() - n0)
        e.close()
    assert counts[1] == counts[0] + 1, counts


# ------------------------------------------------------------------------------------------------- 2. slabs, building blocks
@pytest.mark.parametrize("world", [2, 3])
def test_id_mode_on_slabs_through_the_building_blocks(chd, world):
    """World-many slab engines on one device: border export into device buffers, concatenation, halo import, build, interest
    update, delta.  Entities cross slab borders and are re-homed between ticks (the sender drops them, the receiver adopts them).
    Per rank and slot the delta is the set difference of that rank's visible lists; ids that changed owner or went from halo to
    own (or back) while a slot kept seeing them are in neither list, and the run makes sure that happens."""
    import torch

    wc, x, z, idx = _world(chd, 40_000, 2_000)
    N, S = wc.n_entities, wc.n_subscribers
    radius = 1000.0
    halo = chd.sharding.halo_columns(radius, wc.w)
    cap = N
    # subscribers stand still, each on the rank that owns its column
    cx, cz = x[idx].copy(), z[idx].copy()
    sub_owner = chd.sharding.owner_of_column(chd.sharding.column_of(cx, wc.offx, wc.w, wc.cols), wc.cols, world)
    subs = [np.nonzero(sub_owner == r_)[0] for r_ in range(world)]
    ent_owner = chd.sharding.owner_of_column(chd.sharding.column_of(x, wc.offx, wc.w, wc.cols), wc.cols, world)
    mine = [np.nonzero(ent_owner == r_)[0] for r_ in range(world)]
    engines = []
    for r_ in range(world):
        e = chd.engine.Engine(wc.cfg(), N + cap * world + 16, len(subs[r_]), max_visible=1 << 25)
        lo, hi = chd.sharding.slab_columns(wc.cols, world, r_)
        e.set_slab(lo, hi, halo)
        e.set_subscribers(np.asarray(subs[r_] + 1, np.uint32))
        e.reserve_visible_delta_ids(1 << 22, N)
        engines.append(e)
    recs = [torch.empty(2 * cap, dtype=torch.int32, device="cuda") for _ in range(world)]
    prev = [EMPTY] * world
    prev_own = [set() for _ in range(world)]
    transitions = rehomed = changes = 0
    for t in range(6):
        if t:
            x, z = chd.synth.move_entities(wc, x, z, t, 900.0)
        for r_, e in enumerate(engines):
            e.set_entities(x[mine[r_]], z[mine[r_]])
            e.set_entity_ids(mine[r_].astype(np.uint32))
            assert e.export_border(recs[r_], cap) <= cap
        torch.cuda.synchronize()
        gathered = torch.cat(recs)
        torch.cuda.synchronize()
        for r_, e in enumerate(engines):
            e.import_halo(gathered, cap * world, r_ * cap, cap)
            e.build()
            batch, keep = _batch(chd, np.arange(len(subs[r_])), cx[subs[r_]], cz[subs[r_]], np.full(len(subs[r_]), radius))
            e.update_interest(batch, t * 33 * MS)
            e.visible_delta()
            e.emit_visible()
            s = chd.capi.TickSummary()
            assert chd.capi.lib().chd_summary(e.h, C.byref(s)) == chd.capi.OK and s.overflow == 0
            now = e.get_visible()
            d = e.get_visible_delta()
            _check_delta(d, prev[r_], now)
            if t:
                changes += len(d[1]) + len(d[3])
                # ids a slot saw in both ticks while their ownership on this rank changed
                own_now = set(mine[r_].tolist())
                n = len(subs[r_])
                kept = np.intersect1d(_keys(*prev[r_], n), _keys(*now, n))
                kept_ids = (kept & np.uint64(0xFFFFFFFF)).astype(np.int64)
                flipped = np.fromiter(own_now ^ prev_own[r_], np.int64)
                transitions += int(np.isin(kept_ids, flipped).sum())
            prev[r_], prev_own[r_] = now, set(mine[r_].tolist())
        del gathered
        # re-homing for the next tick: sender drops, receiver adopts
        moves = [e.get_rehome()[:2] for e in engines]
        rehomed += sum(len(g) for g, _ in moves)
        for r_ in range(world):
            leaving = set(moves[r_][0].tolist())
            adopt = [int(g) for (ids, dsts) in moves for g, d_ in zip(ids, dsts) if int(d_) == r_]
            mine[r_] = np.array(sorted((set(mine[r_].tolist()) - leaving) | set(adopt)), np.int64)
    assert changes > 0 and rehomed > 0 and transitions > 0, (changes, rehomed, transitions)
    for e in engines:
        e.close()


# -------------------------------------------------------------------------------------------- 3. chd_tick_sharded at world 1
def test_id_mode_in_tick_sharded_with_migration_at_world_one(chd):
    """chd_tick_sharded with CHD_TICK_VISIBLE_DELTA on a one-rank communicator: every slot's delta is exact, and connections moved
    between slots by chd_migrate_out / chd_migrate_in come out right once netted with sharding.net_migrant_delta."""
    wc, x, z, idx = _world(chd, 30_000, 2_000)
    N, S = wc.n_entities, wc.n_subscribers
    r = np.full(S, 1000.0)
    halo = chd.sharding.halo_columns(1000.0, wc.w)
    cap = N
    e = chd.engine.Engine(wc.cfg(), N + cap + 16, S + 8, max_visible=1 << 25)
    e.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, halo, cap, migrate_subscribers=8, migrate_pairs=8 * 64)
    conn = np.arange(1, S + 1, dtype=np.uint32)
    e.set_subscribers(conn)
    e.reserve_visible_delta_ids(1 << 22, N)
    slot_of = np.arange(S, dtype=np.int64)  # subscriber j -> slot
    migrants = np.array([0, 5, 17], np.int64)
    rng = np.random.default_rng(11)
    prev = EMPTY
    netted = 0
    for t in range(7):
        if t:
            x, z = chd.synth.move_entities(wc, x, z, t, 300.0)
        moved = None
        if t == 3:  # move three connections to fresh slots within the rank
            old, new = slot_of[migrants].copy(), S + np.arange(len(migrants))
            e.migrate_out(old.astype(np.uint32))
            e.migrate_in(0, 0, new.astype(np.uint32), conn[migrants])
            slot_of[migrants] = new
            moved = list(zip(old.tolist(), new.tolist()))
        perm = rng.permutation(N)
        e.set_entities(x[perm], z[perm])
        e.set_entity_ids(perm.astype(np.uint32))
        batch, keep = _batch(chd, slot_of, x[idx], z[idx], r)
        s = e.tick_sharded(batch, (t + 1) * 33 * MS, DELTA_FLAGS)
        assert s.overflow == 0
        now = e.get_visible()
        d = e.get_visible_delta()
        _check_delta(d, prev, now)  # every slot, the vacated and the new ones included
        if moved:
            eo, en, lo, le = d
            for a, b in moved:
                enter, leave = chd.sharding.net_migrant_delta(le[lo[a]:lo[a + 1]], en[eo[b]:eo[b + 1]])
                was = prev[1][prev[0][a]:prev[0][a + 1]]
                sees = now[1][now[0][b]:now[0][b + 1]]
                np.testing.assert_array_equal(np.sort(enter), np.sort(np.setdiff1d(sees, was)))
                np.testing.assert_array_equal(np.sort(leave), np.sort(np.setdiff1d(was, sees)))
                assert len(np.intersect1d(was, sees)) > 0  # the netting cancelled something
                netted += 1
        prev = now
    assert netted == len(migrants)
    assert chd.capi.lib().chd_comm_destroy(e.h) == chd.capi.OK
    e.close()


# -------------------------------------------------------------------------------------------------- 4. errors and overflow
def _summary_tick(chd, e, batch, t, flags=DELTA_FLAGS):
    s = chd.capi.TickSummary()
    st = chd.capi.lib().chd_tick(e.h, C.byref(batch), int(t * 33 * MS), flags, C.byref(s))
    return st, s


@pytest.mark.parametrize("bad", ["out_of_range", "duplicate"])
def test_bad_ids_raise_ovf_delta_ids_and_keep_the_snapshot(chd, bad):
    """An in-world id >= id_space, or one id on two in-world entities: CHD_OVF_DELTA_IDS, no lists, no snapshot advance; the next
    clean delta covers both ticks.  Two entities outside the world sharing an id are not a duplicate."""
    wc, x, z, idx = _world(chd, 20_000, 2_000)
    N, S = wc.n_entities, wc.n_subscribers
    r = np.full(S, wc.radius)
    e = chd.engine.Engine(wc.cfg(), N, S)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta_ids(1 << 22, N)
    ids = np.arange(N, dtype=np.uint32)
    # the last two entities are parked outside the world with the same id: absent, not a duplicate
    x, z = x.copy(), z.copy()
    x[-2:] = wc.offx - 5000.0
    ids_out = ids.copy()
    ids_out[-1] = ids_out[-2]
    e.set_entities(x, z)
    e.set_entity_ids(ids_out)
    batch, keep = _batch(chd, np.arange(S), x[idx], z[idx], r)
    st, s = _summary_tick(chd, e, batch, 0)
    assert st == chd.capi.OK and s.overflow == 0
    base = e.get_visible()
    _check_delta(e.get_visible_delta(), EMPTY, base)
    # tick 1: a bad id on a visible in-world entity
    x1, z1 = chd.synth.move_entities(wc, x, z, 1, 200.0)
    x1[-2:] = wc.offx - 5000.0
    victim = int(idx[10])  # subscriber 10 stands on it: in the world and seen
    bad_ids = ids.copy()
    if bad == "out_of_range":
        bad_ids[victim] = N
    else:
        bad_ids[victim] = bad_ids[int(idx[11])]
    e.set_entities(x1, z1)
    e.set_entity_ids(bad_ids)
    batch, keep = _batch(chd, np.arange(S), x1[idx], z1[idx], r)
    st, s = _summary_tick(chd, e, batch, 1)
    assert st == chd.capi.ERR_CAPACITY and s.overflow == chd.capi.OVF_DELTA_IDS
    with pytest.raises(chd.capi.ChdError) as ei:
        e.get_visible_delta()
    assert ei.value.status == chd.capi.ERR_INVALID
    # tick 2: clean ids again; the delta spans ticks 1 and 2 (the snapshot is still tick 0's)
    x2, z2 = chd.synth.move_entities(wc, x1, z1, 2, 200.0)
    e.set_entities(x2, z2)
    e.set_entity_ids(ids)
    batch, keep = _batch(chd, np.arange(S), x2[idx], z2[idx], r)
    st, s = _summary_tick(chd, e, batch, 2)
    assert st == chd.capi.OK and s.overflow == 0
    now = e.get_visible()
    d = e.get_visible_delta()
    _check_delta(d, base, now)
    assert len(d[1]) + len(d[3]) > 0
    e.close()


def test_ovf_delta_then_reserve_recovers_in_id_mode(chd):
    wc, x, z, idx = _world(chd, 20_000, 2_000)
    N, S = wc.n_entities, wc.n_subscribers
    r = np.full(S, wc.radius)
    e = chd.engine.Engine(wc.cfg(), N, S)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    e.reserve_visible_delta_ids(10, N)  # the first delta enters every visible list: far more than 10
    e.set_entity_ids(np.arange(N, dtype=np.uint32)[::-1].copy())
    e.set_entities(x[::-1].copy(), z[::-1].copy())
    batch, keep = _batch(chd, np.arange(S), x[idx], z[idx], r)
    st, s = _summary_tick(chd, e, batch, 0)
    assert st == chd.capi.ERR_CAPACITY and s.overflow == chd.capi.OVF_DELTA
    ne, nl, ns = e.visible_delta_counts()
    assert ne == s.n_visible and nl == 0 and ns == S
    e.reserve_visible_delta(1 << 22)  # either reserve function only grows the lists of an id-mode engine
    e.reserve_visible_delta_ids(1 << 22, N)
    with pytest.raises(chd.capi.ChdError) as ei:
        e.reserve_visible_delta_ids(1 << 22, N + 1)
    assert ei.value.status == chd.capi.ERR_INVALID
    x1, z1 = chd.synth.move_entities(wc, x, z, 1, 200.0)
    e.set_entities(x1[::-1].copy(), z1[::-1].copy())
    batch, keep = _batch(chd, np.arange(S), x1[idx], z1[idx], r)
    st, s = _summary_tick(chd, e, batch, 1)
    assert st == chd.capi.OK and s.overflow == 0
    _check_delta(e.get_visible_delta(), EMPTY, e.get_visible())
    e.close()
