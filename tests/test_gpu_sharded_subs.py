"""Explicit subscriptions on X-slabs (chd_apply_subscriptions_sharded, include/chd_gpu_subs_sharded.h), against a whole-world engine
that gets the same ops through chd_apply_subscriptions, every tick and per connection: statuses, pairs (cell, dist, interval, flags,
lastFanOutTime, lastMessageIndex), due lists, visible sets and id-mode visible deltas by global id, and the device rings of every
served cell.

The world: 12 x 3 cells of 100 units, halo 2, 3000 entities, slabs on one device joined by the host (border export, halo import,
ring-limit export / import).  Each rank holds regular connections standing in its own columns (half of them send a sphere query every
tick, which diffs explicit pairs away; half never query) and one slot of a "server" connection that subscribes to cells anywhere in
the world: each of its ops goes to the key of the rank that owns the cell's column (sharding.route_sub_ops).
Run on an H100:  python -m pytest tests/test_gpu_sharded_subs.py -m gpu"""
import ctypes as C

import numpy as np
import pytest


pytestmark = pytest.mark.gpu

MS = 1_000_000
COLS, ROWS, W = 12, 3, 100.0
CELLS = COLS * ROWS
HALO = 2
RADIUS = 150.0  # sphere queries reach at most HALO columns beyond the subscriber's own
DEFAULT_IV = 150
N_ENT = 3000
RING_CAP = 2048  # above every ring the floods fill within the longest interval (1000 ms): no CHD_OVF_RING
SERVER = 1000  # the server connection's id
DELTA = 16  # TICK_VISIBLE_DELTA
IVS = np.array([20, 50, 100, 250, 1000], np.uint32)


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
    ns.torch, ns.capi, ns.engine, ns.sharding = torch, capi, engine, sharding
    ns.S0 = engine.SPATIAL_CHANNEL_ID_START
    return ns


def _served_cols(lo, hi):
    col = np.arange(COLS)
    return col[(col + HALO >= lo) & (col < hi + HALO)]


def _batch(chd, slots, cx, cz):
    return chd.engine.make_batch(len(slots), sub=np.asarray(slots, np.uint32),
                                 sphere=(np.asarray(cx, np.float64).copy(), np.asarray(cz, np.float64).copy(), np.full(len(slots), RADIUS)))


def _random_ops(rng, n, keys_cells):
    """n ops on (key, channel) pairs drawn from keys_cells, with every present-bit combination and every option value kind"""
    pick = rng.integers(0, len(keys_cells), n)
    keys = [keys_cells[i][0] for i in pick]
    cell = np.array([keys_cells[i][1] for i in pick], np.int64)
    op = (rng.random(n) < 0.3).astype(np.uint8)
    present = rng.integers(0, 16, n).astype(np.uint8)
    iv = rng.choice(IVS, n)
    dl = rng.integers(-5, 60, n).astype(np.int32)
    ss = rng.integers(0, 2, n).astype(np.uint8)  # SkipSelf = false included
    sf = rng.integers(0, 2, n).astype(np.uint8)
    return keys, cell, op, present, iv, dl, ss, sf


def _apply_whole(chd, whole, slot_of_conn, ops, t):
    keys, cell, op, present, iv, dl, ss, sf = ops
    conn = [k[1] if isinstance(k, tuple) else k for k in keys]
    slots = np.array([slot_of_conn[c] for c in conn], np.uint32)
    return whole.apply_subscriptions(slots, chd.S0 + cell, op, interval=iv, delay=dl, skip_self=ss, skip_first=sf, now_ns=t, present=present)


def _apply_slabs(chd, engines, table, ops, t):
    keys, cell, op, present, iv, dl, ss, sf = ops
    routes = chd.sharding.route_sub_ops(table, keys)
    statuses = []
    for e, (idx, slots) in zip(engines, routes):
        statuses.append(e.apply_subscriptions_sharded(slots, chd.S0 + cell[idx], op[idx], interval=iv[idx], delay=dl[idx], skip_self=ss[idx],
                                                      skip_first=sf[idx], now_ns=t, present=present[idx]))
    return chd.sharding.merge_sub_status(routes, statuses, len(keys))


def _pairs(e, conn_of_slot):
    """sorted (conn, channel, dist, interval, flags, last, last_index) of every pair"""
    p = e.get_pairs()
    slot = np.repeat(np.arange(len(p["off"]) - 1), np.diff(p["off"].astype(np.int64)))
    return sorted((int(conn_of_slot[s]), int(p["channel"][k]), int(p["dist"][k]), int(p["interval"][k]), int(p["flags"][k]), int(p["last"][k]),
                   int(p["last_index"][k])) for k, s in enumerate(slot))


def _dues(e, n_due, conn_of_slot):
    d = e.get_due(n_due)
    return sorted((int(conn_of_slot[x["sub"]]),) + tuple(int(x[k]) for k in d.dtype.names[1:]) for x in d)


def _per_conn(off, ent, conn_of_slot, out=None):
    """conn -> set of ids, merged into `out` (a server's slots on several ranks see disjoint cells)"""
    out = {} if out is None else out
    off = np.asarray(off, np.int64)
    for s in range(len(off) - 1):
        ids = set(np.asarray(ent[off[s]:off[s + 1]]).tolist())
        c = int(conn_of_slot[s])
        assert not (out.get(c, set()) & ids), c
        out.setdefault(c, set()).update(ids)
    return out


def _norm(d):
    return {c: v for c, v in d.items() if v}


class SubWorld:
    """Entities, connections and ops of the module docstring's world for `world` slabs (and a whole-world engine)."""

    def __init__(self, chd, world, seed):
        self.world = world
        self.rng = np.random.default_rng(seed)
        self.x = self.rng.uniform(0, COLS * W, N_ENT)
        self.z = self.rng.uniform(0, ROWS * W, N_ENT)
        self.ent_owner = chd.sharding.owner_of_column(np.floor(self.x / W).astype(np.int64), COLS, world)
        self.table = chd.sharding.SlotTable(world)
        self.cx, self.cz, self.queries = {}, {}, {}
        conn = 1
        for r in range(world):
            lo, hi = chd.sharding.slab_columns(COLS, world, r)
            for k in range(6):
                col = lo + k % (hi - lo)
                self.cx[conn], self.cz[conn] = (col + self.rng.uniform(0.2, 0.8)) * W, self.rng.uniform(0.2, 2.8) * W
                self.queries[conn] = k % 2 == 0
                self.table.place(conn, r)
                conn += 1
        self.regular = list(self.cx)
        for r in range(world):  # the server: one key per rank
            self.table.place(("server", SERVER, r), r)
        self.conn_of_slot = []
        for r in range(world):
            at = self.table.at[r]
            self.conn_of_slot.append(np.array([k[1] if isinstance(k, tuple) else k for _, k in sorted(at.items())], np.uint32))
        self.whole_conns = np.array(self.regular + [SERVER], np.uint32)
        self.whole_slot = {int(c): i for i, c in enumerate(self.whole_conns)}
        # the (key, cell) pairs an op may name: a regular connection's served cells, the server's cells on their column's owner
        self.keys_cells = []
        for c in self.regular:
            lo, hi = chd.sharding.slab_columns(COLS, world, self.table.owner[c])
            for col in _served_cols(lo, hi):
                self.keys_cells += [(c, int(row * COLS + col)) for row in range(ROWS)]
        col_owner = chd.sharding.owner_of_column(np.arange(COLS), COLS, world)
        for cell in range(CELLS):
            self.keys_cells.append((("server", SERVER, int(col_owner[cell % COLS])), cell))
        self.flood = np.zeros(CELLS, bool)
        for r in range(world - 1):  # the columns at each slab border
            hi = chd.sharding.slab_columns(COLS, world, r)[1]
            for col in (hi - 1, hi):
                self.flood[np.arange(ROWS) * COLS + col] = True

    def updates(self, tick, t):
        n = np.where(self.flood, self.rng.integers(100, 151, CELLS) if tick % 2 == 0 else self.rng.integers(50, 101, CELLS),
                     self.rng.integers(0, 9, CELLS))
        off = np.concatenate([[0], np.cumsum(n)]).astype(np.uint32)
        arrival = t - self.rng.integers(0, 5 * MS, int(off[-1])).astype(np.int64)
        sender = self.rng.choice(np.append(self.whole_conns, 77).astype(np.uint32), int(off[-1]))
        return off, arrival, sender

    def query_batch(self, chd, conns, slot_of):
        q = [c for c in conns if self.queries[c]]
        return _batch(chd, [slot_of[c] for c in q], [self.cx[c] for c in q], [self.cz[c] for c in q])


def _ids(table_mode):
    """the entities' global ids: their index, or in entity-table mode index + 1 (id 0 is reserved there)"""
    return np.arange(N_ENT, dtype=np.uint32) + np.uint32(table_mode)


def _make_engines(chd, sw, table_mode, graphs=True):
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    cap = N_ENT
    whole = chd.engine.Engine(cfg, 2 * N_ENT, len(sw.whole_conns), default_fanout_interval_ms=DEFAULT_IV, max_visible=1 << 22)
    if table_mode:
        whole.entity_table_init()
    whole.set_subscribers(sw.whole_conns)
    whole.reserve_visible_delta(1 << 22)
    engines = []
    for r in range(sw.world):
        e = chd.engine.Engine(cfg, 2 * N_ENT + cap * sw.world + 16, len(sw.conn_of_slot[r]), default_fanout_interval_ms=DEFAULT_IV,
                              max_visible=1 << 22)
        e.set_slab(*chd.sharding.slab_columns(COLS, sw.world, r), HALO)
        if table_mode:
            e.entity_table_init()
        e.set_subscribers(sw.conn_of_slot[r])
        e.reserve_visible_delta_ids(1 << 22, N_ENT + 1)
        engines.append(e)
    ids = _ids(table_mode)
    if table_mode:
        assert (whole.spawn_entities(ids, sw.x, sw.z) == 0).all()
        for r, e in enumerate(engines):
            m = sw.ent_owner == r
            assert (e.spawn_entities(ids[m], sw.x[m], sw.z[m]) == 0).all()
    else:
        whole.set_entities(sw.x, sw.z)
    for e in engines + [whole]:
        e.enable_graphs(graphs)
        e.rings_init(RING_CAP)
    return whole, engines


def _exchange_limits(chd, engines, recs):
    import torch

    parts = []
    for e, rec in zip(engines, recs):
        k = e.export_ring_limits(rec, CELLS)
        torch.cuda.synchronize()
        parts.append(rec[:2 * k].clone())
    gathered = torch.cat(parts)
    for e in engines:
        e.import_ring_limits(gathered, len(gathered) // 2)
    return len(gathered) // 2


def _slab_run(chd, world, table_mode, ticks=12):
    import torch

    sw = SubWorld(chd, world, 40 + world + 10 * table_mode)
    whole, engines = _make_engines(chd, sw, table_mode)
    recs = [torch.zeros(2 * CELLS, dtype=torch.int32, device="cuda") for _ in range(world)]
    brec = [torch.empty(2 * N_ENT, dtype=torch.int32, device="cuda") for _ in range(world)]
    ids = _ids(table_mode)
    served = [np.nonzero(np.isin(np.arange(CELLS) % COLS, _served_cols(*chd.sharding.slab_columns(COLS, world, r))))[0] for r in range(world)]
    t = 1000 * MS
    applied = exchanged = dues = diffed = kept = 0
    for tick in range(ticks):
        t += int(sw.rng.integers(90, 131)) * MS
        # 1. the ops, between the ticks
        ops = _random_ops(sw.rng, int(sw.rng.integers(20, 60)), sw.keys_cells)
        want = _apply_whole(chd, whole, sw.whole_slot, ops, t - 7 * MS)
        got = _apply_slabs(chd, engines, sw.table, ops, t - 7 * MS)
        np.testing.assert_array_equal(got, want, err_msg="tick %d statuses" % tick)
        applied += int((want <= chd.capi.SUB_NOT_SUBSCRIBED).sum())
        querying = np.array([sw.queries.get(k, False) for k in ops[0]])  # (a server key is a tuple: it never queries)
        diffed += int(((want == chd.capi.SUB_NEW) & querying).sum())
        # 2. the ring limits the ops (and the last interest updates) raised, then the same updates everywhere
        exchanged += _exchange_limits(chd, engines, recs)
        upd = sw.updates(tick, t)
        for e in engines + [whole]:
            e.rings_append(*upd)
        # 3. the tick
        b, keep = sw.query_batch(chd, sw.regular, sw.whole_slot)
        s = whole.tick(b, t, chd.capi.TICK_ALL | DELTA)
        assert s.overflow == 0
        dues += s.n_due
        w_pairs, w_due = _pairs(whole, sw.whole_conns), _dues(whole, s.n_due, sw.whole_conns)
        w_vis = _norm(_per_conn(*whole.get_visible(), sw.whole_conns))
        eo, en, lo, le = whole.get_visible_delta()
        w_enter, w_leave = _norm(_per_conn(eo, en, sw.whole_conns)), _norm(_per_conn(lo, le, sw.whole_conns))
        W_rings = whole.get_rings()
        if not table_mode:
            for r, e in enumerate(engines):
                m = np.nonzero(sw.ent_owner == r)[0]
                e.set_entities(sw.x[m], sw.z[m])
                e.set_entity_ids(ids[m])
        for r, e in enumerate(engines):
            assert e.export_border(brec[r], N_ENT) <= N_ENT
        torch.cuda.synchronize()
        gathered = torch.cat(brec)
        torch.cuda.synchronize()
        pairs, due, vis, enter, leave = [], [], {}, {}, {}
        for r, e in enumerate(engines):
            e.import_halo(gathered, N_ENT * world, r * N_ENT, N_ENT)
            e.build()
            mine = [c for c in sw.regular if sw.table.owner[c] == r]
            b, keep = sw.query_batch(chd, mine, sw.table.slot)
            s = e.tick(b, t, chd.capi.TICK_EMIT | chd.capi.TICK_FANOUT | DELTA)
            assert s.overflow == 0
            got_rings = e.get_rings()
            for c in served[r]:
                for k in ("arrival", "sender", "index"):
                    np.testing.assert_array_equal(got_rings[k][got_rings["off"][c]:got_rings["off"][c + 1]],
                                                  W_rings[k][W_rings["off"][c]:W_rings["off"][c + 1]], err_msg="tick %d rank %d cell %d" % (tick, r, c))
            np.testing.assert_array_equal(got_rings["msg_index"][served[r]], W_rings["msg_index"][served[r]])
            cos = sw.conn_of_slot[r]
            pairs += _pairs(e, cos)
            due += _dues(e, s.n_due, cos)
            _per_conn(*e.get_visible(), cos, vis)
            eo, en, lo, le = e.get_visible_delta()
            _per_conn(eo, en, cos, enter)
            _per_conn(lo, le, cos, leave)
        del gathered
        assert sorted(pairs) == w_pairs, tick
        assert sorted(due) == w_due, tick
        assert _norm(vis) == w_vis, tick
        assert _norm(enter) == w_enter and _norm(leave) == w_leave, tick
        # a query diffs its slot's explicit pairs away (or keeps them as query pairs); the other slots keep theirs
        assert not [p for p in w_pairs if p[2] == chd.capi.DIST_EXPLICIT and sw.queries.get(p[0], False)], tick
        kept += sum(1 for p in w_pairs if p[2] == chd.capi.DIST_EXPLICIT)
    for e in engines + [whole]:
        e.close()
    assert applied > 100 and dues > 0 and exchanged > 0 and diffed > 0 and kept > 0, (applied, dues, exchanged, diffed, kept)


@pytest.mark.parametrize("table_mode", [False, True], ids=["index", "table"])
@pytest.mark.parametrize("world", [2, 3])
def test_slabs_match_the_whole_world_engine(chd, world, table_mode):
    """12 ticks of random SUB / UNSUB batches between ticks, routed per connection key: every status, pair, due record, visible set,
    visible delta and served ring equals the whole-world engine's for the same connection."""
    _slab_run(chd, world, table_mode)


# ------------------------------------------------------------------------------------------------------------ 2. served range
@pytest.mark.parametrize("world", [2, 3])
def test_outside_slab_exactly_where_the_column_check_says(chd, world):
    """For every cell of the grid, on every rank: a SUB gets OUTSIDE_SLAB exactly where the column lies outside [col_lo - halo,
    col_hi + halo); an UNSUB never does; a bad slot or channel wins over it; a rejected op changes no pair."""
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    for halo in (1, HALO):
        for r in range(world):
            lo, hi = chd.sharding.slab_columns(COLS, world, r)
            e = chd.engine.Engine(cfg, 16, 4)
            e.set_slab(lo, hi, halo)
            e.set_subscribers(np.arange(1, 5, dtype=np.uint32))
            col = np.arange(CELLS) % COLS
            inside = (col + halo >= lo) & (col < hi + halo)
            ch = (chd.S0 + np.arange(CELLS)).astype(np.uint32)
            st = e.apply_subscriptions_sharded(np.zeros(CELLS, np.uint32), ch, np.zeros(CELLS, np.uint8), now_ns=MS)
            np.testing.assert_array_equal(st, np.where(inside, chd.capi.SUB_NEW, chd.capi.SUB_ERR_OUTSIDE_SLAB))
            if lo == 0:
                assert (st[col == 0] == chd.capi.SUB_NEW).all()
            if hi == COLS:
                assert (st[col == COLS - 1] == chd.capi.SUB_NEW).all()
            p = e.get_pairs()
            np.testing.assert_array_equal(p["channel"], ch[inside])
            # UNSUB of every cell: accepted everywhere
            st = e.apply_subscriptions_sharded(np.ones(CELLS, np.uint32), ch, np.ones(CELLS, np.uint8), now_ns=MS)
            assert (st == chd.capi.SUB_NOT_SUBSCRIBED).all()
            # a bad slot, a bad channel, then an outside cell: the first rejection wins
            out = np.nonzero(~inside)[0]
            if len(out):
                c = int(out[0])
                st = e.apply_subscriptions_sharded([9, 1, 1, 2], [chd.S0 + c, chd.S0 + CELLS + 3, chd.S0 - 1, chd.S0 + c], [0, 0, 0, 0], now_ns=MS)
                assert st.tolist() == [chd.capi.SUB_ERR_SLOT, chd.capi.SUB_ERR_CHANNEL, chd.capi.SUB_ERR_CHANNEL, chd.capi.SUB_ERR_OUTSIDE_SLAB]
            q = e.get_pairs()
            for k in p:
                np.testing.assert_array_equal(q[k], p[k])
            e.close()


# ------------------------------------------------------------------------------------------------------------ 3. ring limits
def _raise_run(chd, exchange):
    """Two host-joined slabs; rank 1's connection subscribes explicitly with a 500 ms interval to a flooded cell of rank 0's last
    column (a halo cell of rank 1).  Nothing else raises that cell's limit.  -> ring entries rank 0's replica of the cell differs in."""
    import torch

    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    whole = chd.engine.Engine(cfg, 16, 2, default_fanout_interval_ms=DEFAULT_IV)
    whole.set_subscribers(np.array([1, 2], np.uint32))
    engines = []
    for r in range(2):
        e = chd.engine.Engine(cfg, 16, 1, default_fanout_interval_ms=DEFAULT_IV)
        e.set_slab(*chd.sharding.slab_columns(COLS, 2, r), HALO)
        e.set_subscribers(np.array([r + 1], np.uint32))
        engines.append(e)
    for e in engines + [whole]:
        e.rings_init(RING_CAP)
    cell = 1 * COLS + 5
    recs = [torch.zeros(2 * CELLS, dtype=torch.int32, device="cuda") for _ in range(2)]
    rng = np.random.default_rng(3)
    t = 1000 * MS
    assert whole.apply_subscriptions([1], [chd.S0 + cell], [0], interval=[500], now_ns=t).tolist() == [chd.capi.SUB_NEW]
    assert engines[1].apply_subscriptions_sharded([0], [chd.S0 + cell], [0], interval=[500], now_ns=t).tolist() == [chd.capi.SUB_NEW]
    if exchange:
        assert _exchange_limits(chd, engines, recs) == 1
    differ = 0
    for tick in range(10):
        t += int(rng.integers(90, 131)) * MS
        n = np.zeros(CELLS, np.int64)
        n[cell] = rng.integers(300, 401) if tick % 2 == 0 else rng.integers(150, 201)
        off = np.concatenate([[0], np.cumsum(n)]).astype(np.uint32)
        upd = (off, t - rng.integers(0, 5 * MS, int(off[-1])).astype(np.int64), np.full(int(off[-1]), 9, np.uint32))
        for e in engines + [whole]:
            e.rings_append(*upd)
            assert e.tick(None, t, chd.capi.TICK_FANOUT).overflow == 0
        W_r = whole.get_rings()
        want = W_r["index"][W_r["off"][cell]:W_r["off"][cell + 1]]
        for r, e in enumerate(engines):
            g = e.get_rings()
            got = g["index"][g["off"][cell]:g["off"][cell + 1]]
            if exchange:
                np.testing.assert_array_equal(got, want, err_msg="tick %d rank %d" % (tick, r))
            elif r == 0:
                differ += len(np.setxor1d(got, want))
    for e in engines + [whole]:
        e.close()
    return differ


def test_a_sub_raise_reaches_the_other_ranks_replica(chd):
    """With the exchange after the apply, rank 0's replica of the halo cell keeps what the whole-world ring keeps for the
    subscription (500 ms); skipped, it differs in at least 20 entries: the comparison sees the raise."""
    assert _raise_run(chd, exchange=True) == 0
    assert _raise_run(chd, exchange=False) >= 20


# ---------------------------------------------------------------------------------- 4. chd_tick_sharded at world one, migration
def _comm_world(chd, graphs, migrate=8, rings=True):
    sw = SubWorld(chd, 1, 77)
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    S = len(sw.whole_conns)
    sh = chd.engine.Engine(cfg, 2 * N_ENT + 16, S + migrate, default_fanout_interval_ms=DEFAULT_IV)
    sh.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, HALO, N_ENT, migrate_subscribers=migrate, migrate_pairs=migrate * CELLS)
    one = chd.engine.Engine(cfg, N_ENT, S, default_fanout_interval_ms=DEFAULT_IV)
    for e in (sh, one):
        e.enable_graphs(graphs)
        e.set_subscribers(sw.whole_conns)
        if rings:
            e.rings_init(RING_CAP)
    one.set_entities(sw.x, sw.z)
    return sw, sh, one


@pytest.mark.parametrize("graphs", [True, False])
def test_tick_sharded_with_migration_matches_a_single_engine(chd, graphs):
    """Per tick on a one-rank communicator: chd_tick_sharded; the ops; chd_migrate_out / chd_migrate_in of connections that hold
    explicit pairs of every option kind (to fresh slots, with and without a query in the migration tick; an op on a migrating slot
    gets ERR_SLOT); chd_rings_append; the next chd_tick_sharded.  Pairs, due lists, visible lists and rings equal a single engine's
    per connection on every tick."""
    sw, sh, one = _comm_world(chd, graphs)
    S = len(sw.whole_conns)
    slot_of = dict(sw.whole_slot)  # connection -> slot on sh
    one_conn = sw.whole_conns
    t = 1000 * MS
    moved = 0
    migrants = {3: [1, 2], 6: [3, 4, SERVER]}  # tick -> connections (1, 3: queries; 2, 4, server: none)
    next_slot = S
    for tick in range(10):
        t += int(sw.rng.integers(90, 131)) * MS
        keys_cells = [(c, cell) for c in one_conn.tolist() for cell in range(CELLS)]
        ops = _random_ops(sw.rng, 40, keys_cells)
        if tick in migrants:  # every migrant holds pairs of every option kind before it moves
            for c in migrants[tick]:
                for k, pres in enumerate((0, 1, 2, 4, 8, 15)):
                    ops[0].append(c)
                    ops = (ops[0],) + tuple(np.append(a, v).astype(a.dtype) for a, v in
                                            zip(ops[1:], (3 * k + c % 3, 0, pres, 1000, 25, 0, 1)))
        conns = np.array(ops[0], np.int64)
        args = dict(interval=ops[4], delay=ops[5], skip_self=ops[6], skip_first=ops[7], now_ns=t - 7 * MS, present=ops[3])
        want = one.apply_subscriptions([sw.whole_slot[c] for c in conns], chd.S0 + ops[1], ops[2], **args)
        got = sh.apply_subscriptions_sharded([slot_of[c] for c in conns], chd.S0 + ops[1], ops[2], **args)
        np.testing.assert_array_equal(got, want)
        if tick in migrants:
            ms = migrants[tick]
            old = np.array([slot_of[c] for c in ms], np.uint32)
            new = np.arange(next_slot, next_slot + len(ms), dtype=np.uint32)
            next_slot += len(ms)
            sh.migrate_out(old)
            sh.migrate_in(0, 0, new, np.array(ms, np.uint32))
            st = sh.apply_subscriptions_sharded(np.concatenate([old, new]), np.full(2 * len(ms), chd.S0), np.zeros(2 * len(ms), np.uint8), now_ns=t)
            assert (st == chd.capi.SUB_ERR_SLOT).all()
            for c, s_ in zip(ms, new.tolist()):
                slot_of[c] = s_
            moved += len(ms)
        upd = sw.updates(tick, t)
        for e in (sh, one):
            e.rings_append(*upd)
        sh.set_entities(sw.x, sw.z)
        sh.set_entity_ids(np.arange(N_ENT, dtype=np.uint32))
        b1, k1 = sw.query_batch(chd, sw.regular, slot_of)
        b2, k2 = sw.query_batch(chd, sw.regular, sw.whole_slot)
        s1 = sh.tick_sharded(b1, t, chd.capi.TICK_ALL)
        s2 = one.tick(b2, t, chd.capi.TICK_ALL)
        assert s1.overflow == 0 and s2.overflow == 0
        sh_conn = np.zeros(sh.n_slots, np.uint32)
        for c, s_ in slot_of.items():
            sh_conn[s_] = c
        assert _pairs(sh, sh_conn) == _pairs(one, one_conn), tick
        assert _dues(sh, s1.n_due, sh_conn) == _dues(one, s2.n_due, one_conn), tick
        assert _norm(_per_conn(*sh.get_visible(), sh_conn)) == _norm(_per_conn(*one.get_visible(), one_conn))
        a, b = sh.get_rings(), one.get_rings()
        for k in ("off", "arrival", "sender", "index", "msg_index"):
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    assert moved == 5
    if graphs:
        assert sh.graph_launch_count() > 0
    assert chd.capi.lib().chd_comm_destroy(sh.h) == chd.capi.OK
    for e in (sh, one):
        e.close()


# --------------------------------------------------------------------------------------------------------------------- 5. rules
def test_rules(chd):
    """Refused (CHD_ERR_STATE, nothing changes) on an engine that is not a slab, while a chd_begin_interest is pending and while a
    communicator engine has staged ring updates; accepted after the joining chd_tick / chd_tick_sharded.  chd_apply_subscriptions
    stays refused on a slab."""
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    STATE = chd.capi.ERR_STATE

    def refused(e, fn="apply_subscriptions_sharded"):
        with pytest.raises(chd.capi.ChdError) as ex:
            getattr(e, fn)([0], [chd.S0], [0], now_ns=MS)
        assert ex.value.status == STATE
        assert e.L.chd_apply_subscriptions_sharded(e.h, chd.capi.SubBatch(n=0), 0, None) == (STATE if fn.endswith("sharded") else chd.capi.OK)

    plain = chd.engine.Engine(cfg, 16, 4)
    plain.set_subscribers(np.arange(1, 5, dtype=np.uint32))
    refused(plain)
    plain.close()
    slab = chd.engine.Engine(cfg, 16, 4)
    slab.set_slab(0, 6, HALO)
    slab.rings_init(RING_CAP)
    slab.set_subscribers(np.arange(1, 5, dtype=np.uint32))
    refused(slab, "apply_subscriptions")
    b, keep = _batch(chd, [1], [50.0], [50.0])
    slab.begin_interest(b, MS)
    refused(slab)
    slab.tick(None, MS, chd.capi.TICK_FANOUT)
    assert slab.apply_subscriptions_sharded([0], [chd.S0], [0], now_ns=2 * MS).tolist() == [chd.capi.SUB_NEW]
    p = slab.get_pairs()
    assert p["off"][1] == 1 and p["channel"][0] == chd.S0 and p["dist"][0] == chd.capi.DIST_EXPLICIT and p["off"][2] > 1
    slab.close()
    sw, sh, one = _comm_world(chd, True)
    upd = sw.updates(0, 1000 * MS)
    sh.rings_append(*upd)
    refused(sh)
    sh.set_entities(sw.x, sw.z)
    sh.set_entity_ids(np.arange(N_ENT, dtype=np.uint32))
    sh.tick_sharded(None, 1000 * MS, chd.capi.TICK_ALL)
    assert sh.apply_subscriptions_sharded([0], [chd.S0 + 7], [0], now_ns=1001 * MS).tolist() == [chd.capi.SUB_NEW]
    assert chd.capi.lib().chd_comm_destroy(sh.h) == chd.capi.OK
    for e in (sh, one):
        e.close()


def test_capacity_is_transactional_per_rank(chd):
    """A batch that would take a slab past max_pairs applies nothing there: every valid op gets ERR_CAPACITY, the summary carries
    CHD_OVF_PAIRS and required_pairs, the pairs are unchanged; OUTSIDE_SLAB and ERR_SLOT keep their statuses."""
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    e = chd.engine.Engine(cfg, 16, 4, max_pairs=16)
    e.set_slab(0, 6, HALO)  # serves columns 0-7
    e.set_subscribers(np.arange(1, 5, dtype=np.uint32))
    assert (e.apply_subscriptions_sharded([0, 1, 2], chd.S0 + np.arange(3), [0, 0, 0], now_ns=MS) == chd.capi.SUB_NEW).all()
    before = e.get_pairs()
    cells = [3, 4, 5, 6, 7] + list(range(12, 20)) + [24]  # 14 served cells: 17 pairs > 16
    slots = np.array([0] * 14 + [3, 9], np.uint32)
    ch = (chd.S0 + np.array(cells + [11, 1])).astype(np.uint32)
    st = e.apply_subscriptions_sharded(slots, ch, np.zeros(16, np.uint8), now_ns=2 * MS)
    assert st.tolist() == [chd.capi.SUB_ERR_CAPACITY] * 14 + [chd.capi.SUB_ERR_OUTSIDE_SLAB, chd.capi.SUB_ERR_SLOT]
    with pytest.raises(chd.capi.ChdError):  # CHD_OVF_PAIRS (the summary reads and clears the bit)
        e.summary()
    s = chd.capi.TickSummary()
    assert e.L.chd_summary(e.h, C.byref(s)) == chd.capi.OK and s.n_pairs == 3 and s.required_pairs == 17
    after = e.get_pairs()
    for k in before:
        np.testing.assert_array_equal(after[k], before[k])
    e.close()


def test_ticks_without_the_feature_launch_the_same(chd):
    """chd_tick_sharded launches the same kernels and graphs whether or not explicit ops were applied before it."""
    counts = []
    for with_ops in (False, True):
        sw, sh, one = _comm_world(chd, True, rings=False)
        b, keep = sw.query_batch(chd, sw.regular, sw.whole_slot)
        sh.set_entities(sw.x, sw.z)
        sh.set_entity_ids(np.arange(N_ENT, dtype=np.uint32))
        for k in range(6):  # warm-up: both pair-buffer parities captured
            sh.tick_sharded(b, (k + 1) * 33 * MS, chd.capi.TICK_ALL)
        if with_ops:
            sh.apply_subscriptions_sharded([0, 1, 2], chd.S0 + np.array([1, 2, 3]), [0, 0, 0], now_ns=7 * 33 * MS)
            sh.apply_subscriptions_sharded([0], [chd.S0 + 9], [0], now_ns=7 * 33 * MS)
        l0, g0 = sh.launch_count(), sh.graph_launch_count()
        for k in range(6, 14):
            sh.tick_sharded(b, (k + 1) * 33 * MS, chd.capi.TICK_ALL)
        counts.append((sh.launch_count() - l0, sh.graph_launch_count() - g0))
        assert chd.capi.lib().chd_comm_destroy(sh.h) == chd.capi.OK
        for e in (sh, one):
            e.close()
    assert counts[0] == counts[1], counts
