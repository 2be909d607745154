"""Device-owned update rings on X-slabs (include/chd_gpu_rings.h): every rank keeps a replica of the ring of each cell it serves,
fed the same whole-grid updates, and evicts by maxFanOutIntervalMs exchanged as ring-limit records, so that every replica equals the
ring of one whole-world engine fed the same updates and queries.  Checked every tick, for every served cell, against that engine:
every ring entry and msgIndex, the due list and the committed pair state of the rank's subscribers.

The world (`RingWorld`): 12 x 3 cells of 100 units, split into slabs; each slab but the last floods its three rightmost columns
with 150-400 updates a tick (even ticks 300-400, odd ticks 150-200) and watches them at dist 0 (20 ms), and each slab but the
first watches them from its leftmost column at dist 1-3 (50, 100 ms and the default interval, 150 ms here) from tick 2 on.  The
cell's maximum therefore lives on the right-hand neighbour only.  Ticks:
  cap 620  gaps of 90-130 ms: the previous tick's flood is younger than 150 ms, so the whole-world ring grows above 512 (to at most
           the last two floods, 600) where a slab that evicts by its own 20 ms does not.  The same run without the ring-limit
           calls differs in its replicas, which shows that the comparison sees a missing exchange.
  cap 513  gaps of 170-260 ms: a ring above 512 must evict on every append (a slab of 513 has no room to grow), so every older
           flood is evictable; the rings slide back to their slab start on almost every tick.
Run on an H100:  python -m pytest tests/test_gpu_sharded_rings.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_rings_scale import _status

pytestmark = pytest.mark.gpu

MS = 1_000_000
COLS, ROWS, W = 12, 3, 100.0
DEFAULT_IV = 150  # default_fanout_interval_ms: the interval of dist >= 3
HALO = 4
FAR_FROM = 2  # the tick from which the far subscribers reach across the border
GAPS_MS = {620: (100, 95, 120, 90, 110, 130, 100, 95, 115, 105), 513: (170, 185, 240, 170, 200, 175, 260, 180, 190, 175)}


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
    return ns


class RingWorld:
    """Subscribers and updates of the module docstring's world, laid out for `split` slabs (whoever hosts them)."""

    def __init__(self, split, cap, seed):
        self.split, self.cap = split, cap
        self.rng = np.random.default_rng(seed)
        self.cells = COLS * ROWS
        self.hot = np.zeros(self.cells, bool)
        # per pseudo-rank: subscriber centres and (early, late) radii
        self.subs = []
        for r in range(split):
            lo, hi = r * COLS // split, (r + 1) * COLS // split
            cx, cz, r0, r1 = [], [], [], []
            for row in range(ROWS):
                if r < split - 1:
                    for col in range(hi - 3, hi):
                        self.hot[row * COLS + col] = True
                        cx.append((col + 0.5) * W), cz.append((row + 0.5) * W), r0.append(0.2 * W), r1.append(0.2 * W)
                if r > 0:
                    cx.append((lo + 0.5) * W), cz.append((row + 0.5) * W), r0.append(0.2 * W), r1.append(3.3 * W)
            self.subs.append(tuple(np.array(a) for a in (cx, cz, r0, r1)))
        self.conn = []
        k = 1
        for s in self.subs:
            self.conn.append(np.arange(k, k + len(s[0]), dtype=np.uint32))
            k += len(s[0])
        self.t = 1000 * MS

    def times(self):
        out, t = [], self.t
        for g in GAPS_MS[self.cap]:
            t += g * MS
            out.append(t)
        return out

    def queries(self, ranks, tick):
        """sphere arrays of the subscribers of `ranks`, in conn order"""
        cx = np.concatenate([self.subs[r][0] for r in ranks])
        cz = np.concatenate([self.subs[r][1] for r in ranks])
        rad = np.concatenate([self.subs[r][3 if tick >= FAR_FROM else 2] for r in ranks])
        return cx, cz, rad

    def updates(self, tick, t):
        n = np.where(self.hot, self.rng.integers(300, 401, self.cells) if tick % 2 == 0 else self.rng.integers(150, 201, self.cells),
                     self.rng.integers(0, 9, self.cells))
        off = np.concatenate([[0], np.cumsum(n)]).astype(np.uint32)
        arrival = t - self.rng.integers(0, 5 * MS, int(off[-1])).astype(np.int64)
        sender = self.rng.integers(1, int(self.conn[-1][-1]) + 1, int(off[-1])).astype(np.uint32)
        return off, arrival, sender


def _batch(chd, cx, cz, rad):
    return chd.engine.make_batch(len(cx), sub=np.arange(len(cx), dtype=np.uint32), sphere=(cx.copy(), cz.copy(), rad.copy()))


def _served(lo, hi):
    col = np.arange(COLS * ROWS) % COLS
    return np.nonzero((col + HALO >= lo) & (col < hi + HALO))[0]


def _cell_rings(R):
    off = R["off"].astype(np.int64)
    return {c: (R["arrival"][off[c]:off[c + 1]], R["sender"][off[c]:off[c + 1]], R["index"][off[c]:off[c + 1]]) for c in range(len(off) - 1)}


def _assert_rings_on(got, want, cells, what):
    g, w = _cell_rings(got), _cell_rings(want)
    for c in cells:
        for k in range(3):
            np.testing.assert_array_equal(g[c][k], w[c][k], err_msg="%s cell %d" % (what, c))
    np.testing.assert_array_equal(got["msg_index"][cells], want["msg_index"][cells], err_msg=what)


def _ring_difference(got, want, cells):
    """entries in one ring and not in the other (by message index), over `cells`"""
    g, w = _cell_rings(got), _cell_rings(want)
    return sum(len(np.setxor1d(g[c][2], w[c][2])) for c in cells)


def _due_set(e, n_due, conn_of_slot):
    d = e.get_due(n_due)
    return {(int(conn_of_slot[x["sub"]]),) + tuple(int(x[k]) for k in d.dtype.names[1:]) for x in d}


def _pair_set(e, conn_of_slot):
    p = e.get_pairs()
    slot = np.repeat(np.arange(len(p["off"]) - 1), np.diff(p["off"].astype(np.int64)))
    return {(int(conn_of_slot[s]), int(p["channel"][k]), int(p["dist"][k]), int(p["interval"][k]), int(p["flags"][k]), int(p["last"][k]),
             int(p["last_index"][k])) for k, s in enumerate(slot)}


def _slab_run(chd, world, cap, exchange, graphs=True):
    """World-many slab engines on one device next to a whole-world engine.  Per tick: every slab imports every record of the last
    exports (exchange), every engine appends the same updates, ticks (interest update + fan-out) and every slab exports.  -> the number
    of ring entries the replicas differ from the whole-world rings in, over their served cells (0 when everything matched)."""
    import torch

    rw = RingWorld(world, cap, 11 + world)
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    S = sum(len(c) for c in rw.conn)
    whole = chd.engine.Engine(cfg, 16, S, default_fanout_interval_ms=DEFAULT_IV)
    whole.set_subscribers(np.concatenate(rw.conn))
    engines, served = [], []
    for r in range(world):
        lo, hi = chd.sharding.slab_columns(COLS, world, r)
        e = chd.engine.Engine(cfg, 16, len(rw.conn[r]), default_fanout_interval_ms=DEFAULT_IV)
        e.set_slab(lo, hi, HALO)
        e.set_subscribers(rw.conn[r])
        engines.append(e)
        served.append(_served(lo, hi))
    for e in engines + [whole]:
        e.enable_graphs(graphs)
        e.rings_init(cap)
    rec_cap = max(len(s) for s in served)
    recs = [torch.zeros(2 * rec_cap, dtype=torch.int32, device="cuda") for _ in range(world)]
    gathered, n_gathered = None, 0
    differ = capacity_checked = raised = n_due = 0
    for tick, t in enumerate(rw.times()):
        upd = rw.updates(tick, t)
        if exchange and n_gathered:
            for e in engines:
                e.import_ring_limits(gathered, n_gathered)
        whole.rings_append(*upd)
        sw = whole.tick(_batch(chd, *rw.queries(range(world), tick))[0], t, chd.capi.TICK_FANOUT)
        assert sw.overflow == 0
        n_due += sw.n_due
        W_rings = whole.get_rings()
        conn_all = np.concatenate(rw.conn)
        w_due, w_pairs = _due_set(whole, sw.n_due, conn_all), _pair_set(whole, conn_all)
        for r, e in enumerate(engines):
            e.rings_append(*upd)
            b, keep = _batch(chd, *rw.queries([r], tick))
            s = e.tick(b, t, chd.capi.TICK_FANOUT)
            assert s.overflow == 0
            got = e.get_rings()
            if not exchange:
                differ += _ring_difference(got, W_rings, served[r])
                continue
            _assert_rings_on(got, W_rings, served[r], "tick %d rank %d" % (tick, r))
            mine = set(rw.conn[r].tolist())
            assert _due_set(e, s.n_due, rw.conn[r]) == {x for x in w_due if x[0] in mine}, (tick, r)
            assert _pair_set(e, rw.conn[r]) == {x for x in w_pairs if x[0] in mine}, (tick, r)
        if not exchange:
            continue
        parts = []
        for r, e in enumerate(engines):
            n = C.c_uint32()
            p = chd.capi.ptr(recs[r])
            st = e.L.chd_export_ring_limits(e.h, p, 0, C.byref(n))  # how many: refused, nothing advanced
            k = n.value
            assert st == (chd.capi.ERR_CAPACITY if k else chd.capi.OK)
            if k:
                assert e.L.chd_export_ring_limits(e.h, p, k - 1, C.byref(n)) == chd.capi.ERR_CAPACITY and n.value == k
                capacity_checked += 1
            assert e.export_ring_limits(recs[r], rec_cap) == k  # the same raises, now exported
            assert e.export_ring_limits(recs[r], rec_cap) == 0  # ... and marked
            raised += k
            torch.cuda.synchronize()
            parts.append(recs[r][:2 * k].clone())
        gathered = torch.cat(parts)
        n_gathered = len(gathered) // 2
    for e in engines + [whole]:
        e.close()
    assert n_due > 0
    if exchange:
        assert capacity_checked > 0 and raised > 0
    return differ


@pytest.mark.parametrize("cap", [513, 620])
@pytest.mark.parametrize("world", [2, 3])
def test_slab_replicas_match_the_whole_world_rings(chd, world, cap):
    """With the ring-limit exchange every rank's rings, msgIndex, due list and pairs equal the whole-world engine's on its served
    cells every tick.  At cap 620 the same run without the exchange differs (the slab that holds the near subscribers evicts by
    20 ms where the whole world keeps the far subscribers' 150 ms): the comparison sees a missing exchange, and slabs that do
    not exchange keep evicting by their own maximum."""
    assert _slab_run(chd, world, cap, exchange=True) == 0
    if cap == 620:
        assert _slab_run(chd, world, cap, exchange=False) >= 20


def test_slab_refusals(chd):
    """Ring limits need device rings on a slab, and go before a chd_begin_interest."""
    import torch

    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    rec = torch.zeros(2 * COLS * ROWS, dtype=torch.int32, device="cuda")
    plain = chd.engine.Engine(cfg, 16, 4)
    plain.rings_init(513)
    slab = chd.engine.Engine(cfg, 16, 4)
    slab.set_slab(0, 6, HALO)
    for e in (plain, slab):  # no slab / no device rings
        for st in (e.L.chd_export_ring_limits(e.h, chd.capi.ptr(rec), COLS * ROWS, None), e.L.chd_import_ring_limits(e.h, chd.capi.ptr(rec), 1)):
            assert st == chd.capi.ERR_STATE
    slab.rings_init(513)
    slab.set_subscribers(np.arange(1, 5, dtype=np.uint32))
    b, keep = _batch(chd, np.full(4, 50.0), np.full(4, 50.0), np.full(4, 20.0))
    slab.begin_interest(b, MS)
    assert slab.L.chd_export_ring_limits(slab.h, chd.capi.ptr(rec), COLS * ROWS, None) == chd.capi.ERR_STATE
    assert slab.L.chd_import_ring_limits(slab.h, chd.capi.ptr(rec), 1) == chd.capi.ERR_STATE
    slab.tick(None, MS, chd.capi.TICK_FANOUT)
    assert slab.export_ring_limits(rec, COLS * ROWS) == 1  # the one cell the update raised
    for e in (plain, slab):
        e.close()


# ------------------------------------------------------------------------------------------------- chd_tick_sharded at world one
def _world_one(chd, graphs, n_ent=3000):
    rw = RingWorld(2, 620, 5)
    cfg = chd.engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    S = sum(len(c) for c in rw.conn)
    rng = np.random.default_rng(6)
    x, z = rng.uniform(0, COLS * W, n_ent), rng.uniform(0, ROWS * W, n_ent)
    sh = chd.engine.Engine(cfg, 2 * n_ent + 16, S, default_fanout_interval_ms=DEFAULT_IV)
    one = chd.engine.Engine(cfg, n_ent, S, default_fanout_interval_ms=DEFAULT_IV)
    sh.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, HALO, n_ent)
    conn = np.concatenate(rw.conn)
    for e in (sh, one):
        e.enable_graphs(graphs)
        e.set_subscribers(conn)
        e.rings_init(620)
    return rw, sh, one, conn, x, z


def _compare(chd, sh, one, s1, s2, conn):
    assert s1.overflow == 0 and s2.overflow == 0 and s1.n_due == s2.n_due
    a, b = sh.get_rings(), one.get_rings()
    for k in ("off", "arrival", "sender", "index", "msg_index"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    assert _due_set(sh, s1.n_due, conn) == _due_set(one, s2.n_due, conn)
    assert _pair_set(sh, conn) == _pair_set(one, conn)
    for u, v in zip(sh.get_visible(), one.get_visible()):
        np.testing.assert_array_equal(u, v)


@pytest.mark.parametrize("graphs", [True, False])
def test_tick_sharded_with_device_rings_at_world_one_matches_a_single_engine(chd, graphs):
    """chd_tick_sharded on a one-rank communicator with device rings: chd_rings_append stages the updates, the tick exchanges the
    ring limits with itself, appends and then updates the interest.  The rings, msgIndex, due list, pairs and visible lists equal a
    plain engine's driven by chd_rings_append + chd_tick, on every tick."""
    rw, sh, one, conn, x, z = _world_one(chd, graphs)
    for tick, t in enumerate(rw.times()[:8]):
        upd = rw.updates(tick, t)
        b, keep = _batch(chd, *rw.queries([0, 1], tick))
        sh.set_entities(x, z)
        sh.set_entity_ids(np.arange(len(x), dtype=np.uint32))
        one.set_entities(x, z)
        for e in (sh, one):
            e.rings_append(*upd)
        s1 = sh.tick_sharded(b, t, chd.capi.TICK_ALL)
        s2 = one.tick(b, t, chd.capi.TICK_ALL)
        _compare(chd, sh, one, s1, s2, conn)
    if graphs:
        assert sh.graph_launch_count() > 0
    assert chd.capi.lib().chd_comm_destroy(sh.h) == chd.capi.OK
    for e in (sh, one):
        e.close()


def test_staged_updates_on_a_communicator_engine(chd):
    """One chd_rings_append per tick on a communicator engine: while its updates are staged, a second append and chd_get_rings,
    chd_tick, chd_begin_interest and chd_update_interest are refused and change nothing; the next chd_tick_sharded applies the
    staged updates once (the rings then equal a plain engine's that appended them once).  With device rings, chd_tick_sharded
    refuses a host's pending chd_begin_interest."""
    rw, sh, one, conn, x, z = _world_one(chd, True)
    L, OK, STATE = sh.L, chd.capi.OK, chd.capi.ERR_STATE
    times = rw.times()
    for tick in range(3):
        upd = rw.updates(tick, times[tick])
        b, keep = _batch(chd, *rw.queries([0, 1], tick))
        sh.set_entities(x, z)
        sh.set_entity_ids(np.arange(len(x), dtype=np.uint32))
        one.set_entities(x, z)
        if tick == 2:  # a host's own chd_begin_interest: not with device rings
            sh.begin_interest(b, times[tick])
            assert L.chd_tick_sharded(sh.h, None, times[tick], chd.capi.TICK_ALL, None) == STATE
            sh.tick(None, times[tick], chd.capi.TICK_ALL)  # (joins it)
            break
        one.rings_append(*upd)
        sh.rings_append(*upd)
        if tick == 1:
            other = rw.updates(tick, times[tick])  # (a different batch: applying it would show)
            assert _status(lambda: sh.rings_append(*other)) == STATE
            assert _status(sh.get_rings) == STATE
            assert L.chd_tick(sh.h, C.byref(b), times[tick], chd.capi.TICK_ALL, None) == STATE
            assert L.chd_begin_interest(sh.h, C.byref(b), times[tick], 1) == STATE
            assert L.chd_update_interest(sh.h, C.byref(b), times[tick]) == STATE
            assert "staged" in L.chd_last_error(sh.h).decode()
        s1 = sh.tick_sharded(b, times[tick], chd.capi.TICK_ALL)
        s2 = one.tick(b, times[tick], chd.capi.TICK_ALL)
        _compare(chd, sh, one, s1, s2, conn)
    assert chd.capi.lib().chd_comm_destroy(sh.h) == OK
    for e in (sh, one):
        e.close()
