"""Device-owned update rings (chd_rings_init / chd_rings_append / chd_get_rings: the buffer half of ChannelData.OnUpdate,
data.go:149-173) and the fan-out over them, against the oracle's channels (one per cell) fed the same subscriptions and updates.

Each cell owns a slab of `cap` entries; its live ring is [begin, end) inside it, the tail slides back to the slab start when it
reaches the slab end, and a slab full of live entries drops its oldest one (CHD_OVF_RING).  The fan-out stages a block's ring
span begin[first cell] .. end[last cell] in shared memory when it holds at most FANOUT_STAGE entries: over slabs that span crosses
the dead space between live rings.  `_Slabs` restates where begin / end go; it is used only to assert that each case takes the
paths it is named for:
  grid  cells   slab cap            paths asserted
  a     225     513, 1024           evictions (one where a kept pair's interval is above its channel's maximum), slides, pairs with
  b     300     513, 1024 (+ start  more than FANOUT_SLOTS decisions, multi-cell blocks on the global path (and the staged one at
  e     65536   times), 620         cap 513); 620: multi-cell block spans of exactly 640 (staged) and 641 (global)
plus the same world through chd_tick(TICK_ALL) with graphs on and off and in the pipelined loop, a full slab, the argument edges,
and the call order: ring inputs are refused while a chd_begin_interest is pending.
Run on an H100:  python -m pytest tests/test_gpu_rings_scale.py -m gpu
"""
import ctypes as C
from collections import deque

import numpy as np
import pytest

from tests.test_gpu_fanout_scale import FANOUT_BLOCK, FANOUT_STAGE, _due_table, _intervals, _pair_keys

pytestmark = pytest.mark.gpu

S0 = 65536
MS = 1_000_000
MAX_BUFFER = 512  # MaxUpdateMsgBufferSize (data.go:53-55)
GRIDS = {  # offx, offz, w, h, cols, rows
    "a": (-15000.0, -15000.0, 2000.0, 2000.0, 15, 15),
    "b": (-1000.0, -750.0, 100.0, 100.0, 20, 15),
    "e": (-12800.0, -12800.0, 100.0, 100.0, 256, 256),
}
RADII = {"a": (50.0, 1500.0, 2500.0)}
# irregular ticks, every gap above the longest interval (100 ms) plus the spread of a flood's arrivals: once a flooded buffer holds
# more than 512 entries its oldest one is always older than maxFanOutIntervalMs, so the buffer never outgrows a 513-entry slab
GAPS_MS = (110, 125, 240, 110, 180, 130, 260, 115)
FLOOD_SPREAD_NS = 5 * MS
N_TICKS = len(GAPS_MS)
N_SPECIAL = 4  # subscribers that alone watch cell D: created at dist 0 (20 ms), moved to dist 2 (100 ms) from tick 2 on

CASES = [pytest.param(g, cap, False, id="%s-cap%d" % (g, cap)) for g in ("a", "b", "e") for cap in (513, 1024)]
CASES += [pytest.param("b", 1024, True, id="b-cap1024-starts"), pytest.param("b", 620, False, id="b-stage")]


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
    ns.torch, ns.capi, ns.engine = torch, capi, engine
    return ns


def _status(f):
    """an Engine method's status (it raises ChdError on anything but OK)"""
    from channeld_b200.capi import OK, ChdError

    try:
        f()
    except ChdError as ex:
        return ex.status
    return OK


def _assert_rings(got, want, skip=()):
    """the device rings equal the oracle's buffers, cell by cell except the cells in `skip`"""
    g_len, w_len = np.diff(got["off"].astype(np.int64)), np.diff(want["off"].astype(np.int64))
    keep = np.ones(len(g_len), bool)
    keep[list(skip)] = False
    np.testing.assert_array_equal(g_len[keep], w_len[keep])
    np.testing.assert_array_equal(got["msg_index"], want["msg_index"])
    gm, wm = np.repeat(keep, g_len), np.repeat(keep, w_len)
    for k in ("arrival", "sender", "index"):
        np.testing.assert_array_equal(got[k][gm], want[k][wm], err_msg=k)


def _csr(n_cell):
    return np.concatenate([[0], np.cumsum(n_cell)]).astype(np.uint32)


class _Slabs:
    """Where each cell's live ring sits in its slab (rings_append_kernel's slide and drop rules), from the oracle's buffers: for
    the path assertions only."""

    def __init__(self, cells, cap):
        self.cap = cap
        self.b = np.zeros(cells, np.int64)
        self.e = np.zeros(cells, np.int64)
        self.evictions = np.zeros(cells, np.int64)
        self.slides = np.zeros(cells, np.int64)
        self.drops = np.zeros(cells, np.int64)

    def append(self, n_cell, u_arr, before, max_iv):
        """n_cell updates per cell (arrivals u_arr, CSR by cell), `before` = the oracle's buffers just before them.  -> evictions
        per cell"""
        cap, b, e = self.cap, self.b, self.e
        n_cell = np.asarray(n_cell, np.int64)
        live = e - b
        # a cell whose buffer stays within 512 and whose tail does not reach the slab end only moves its tail
        easy = (live + n_cell <= MAX_BUFFER) & (e + n_cell <= cap)
        e[easy] += n_cell[easy]
        ev = np.zeros(len(n_cell), np.int64)
        u_off, r_off = _csr(n_cell).astype(np.int64), before["off"].astype(np.int64)
        for c in np.nonzero(~easy)[0]:
            ring = deque(before["arrival"][r_off[c]:r_off[c + 1]].tolist())
            assert len(ring) == live[c]
            bc, ec, mx = int(b[c]), int(e[c]), int(max_iv[c]) * MS
            for t in u_arr[u_off[c]:u_off[c + 1]].tolist():
                if ec == cap:
                    n = ec - bc
                    if n == cap:
                        self.drops[c] += 1
                        ring.popleft()
                        n -= 1
                    self.slides[c] += 1
                    bc, ec = 0, n
                ring.append(t)
                ec += 1
                if ec - bc > MAX_BUFFER and ring[0] + mx < t:
                    ring.popleft()
                    bc += 1
                    ev[c] += 1
            b[c], e[c] = bc, ec
        self.evictions += ev
        return ev

    def block_spans(self, cell_sorted):
        """ring span (end[last cell] - begin[first cell], slab-laid) of every fan-out block and whether it covers several cells"""
        cap = self.cap
        lo = cell_sorted[::FANOUT_BLOCK]
        hi = cell_sorted[FANOUT_BLOCK - 1::FANOUT_BLOCK]
        if len(hi) < len(lo):
            hi = np.concatenate([hi, cell_sorted[-1:]])
        return (hi * cap + self.e[hi]) - (lo * cap + self.b[lo]), hi > lo


class _World:
    """100 K subscribers on a grid, moving, with mixed sphere radii; cell D is watched only by N_SPECIAL subscribers, created at
    dist 0 and moved to dist 2 (a kept pair whose interval rises above its channel's maxFanOutIntervalMs).  Hot cells (D among
    them) get 150-400 updates a tick, the others 0-8; arrivals are not time-sorted, half the senders are subscribed to the cell."""

    def __init__(self, oracle, grid, seed, n_sub=100_000, n_hot=12, stage=False, starts=False):
        from tests._oracle import make_grid

        self.g = GRIDS[grid]
        offx, offz, w, h, cols, rows = self.g
        self.og = make_grid(*self.g)
        self.C = C_ = cols * rows
        self.W, self.H = w * cols, h * rows
        self.rng = rng = np.random.default_rng(seed)
        self.S = n_sub
        self.conn = np.arange(1, n_sub + 1, dtype=np.uint32)
        radii = RADII.get(grid, (50.0, 60.0, 120.0))
        self.rad = rng.choice(radii, n_sub)
        dc, dr = cols // 2, rows // 2
        self.D = dr * cols + dc
        self.zone = int(np.ceil(max(radii) / w)) + 1  # a subscriber centred further away cannot reach D
        self.dx, self.dz = offx + (dc + 0.5) * w, offz + (dr + 0.5) * h
        # queries of the special subscribers (searched with the oracle: D at dist 0, then at dist 2)
        self.q_near = (self.dx, self.dz, 0.2 * w)
        self.q_far = (self.dx + 2 * w, self.dz, 2.0 * w)
        for q, d in ((self.q_near, 0), (self.q_far, 2)):
            res, st = oracle.query(self.og, sphere=q)
            assert st == 0 and res[S0 + self.D] == d
        self.cx, self.cz = self._outside(offx + rng.random(n_sub) * self.W, offz + rng.random(n_sub) * self.H)
        self.stage = stage
        self.hot = np.zeros(C_, bool)
        if not stage:
            self.hot[rng.choice(np.setdiff1d(np.arange(C_), [self.D]), n_hot, replace=False)] = True
            self.hot[self.D] = True
        self.start = (np.arange(C_) % 4 * 250 * MS).astype(np.int64) if starts else None
        self.t = 1000 * MS

    def _in_zone(self, x, z):
        offx, offz, w, h, cols, rows = self.g
        ci = np.floor((x - offx) / w).astype(np.int64) - self.D % cols
        ri = np.floor((z - offz) / h).astype(np.int64) - self.D // cols
        return np.maximum(np.abs(ci), np.abs(ri)) <= self.zone

    def _outside(self, x, z):
        offx, offz = self.g[0], self.g[1]
        while True:
            bad = self._in_zone(x, z)
            if not bad.any():
                return x, z
            x[bad] = offx + self.rng.random(bad.sum()) * self.W
            z[bad] = offz + self.rng.random(bad.sum()) * self.H

    def next_tick(self, tick):
        """advances the clock and the subscribers -> (t, cx, cz, rad) of this tick's queries (every subscriber sends one)"""
        offx, offz, w, h = self.g[:4]
        rng = self.rng
        self.t += GAPS_MS[tick] * MS
        if tick:
            mv = rng.random(self.S) < 0.3
            nx = np.clip(self.cx + rng.uniform(-0.6, 0.6, self.S) * w * mv, offx + 1e-3, offx + self.W - 1e-3)
            nz = np.clip(self.cz + rng.uniform(-0.6, 0.6, self.S) * h * mv, offz + 1e-3, offz + self.H - 1e-3)
            stay = self._in_zone(nx, nz)
            self.cx, self.cz = np.where(stay, self.cx, nx), np.where(stay, self.cz, nz)
        cx, cz, rad = self.cx.copy(), self.cz.copy(), self.rad.copy()
        q = self.q_near if tick < 2 else self.q_far
        cx[-N_SPECIAL:], cz[-N_SPECIAL:], rad[-N_SPECIAL:] = q
        return self.t, cx, cz, rad

    def updates(self, tick, w_sub, w_cell):
        """this tick's updates, CSR by cell -> (n_cell, arrival (channel time), sender)"""
        rng, C_, t = self.rng, self.C, self.t
        if self.stage:  # plain cells only: every live ring starts at its slab start and holds at most 64 entries
            n_cell = rng.integers(0, 9, C_)
        else:
            n_cell = np.where(self.hot, rng.integers(150, 401, C_), rng.integers(0, 9, C_))
        n = int(n_cell.sum())
        u_cell = np.repeat(np.arange(C_), n_cell)
        hot = self.hot[u_cell]
        spread = np.where(hot, FLOOD_SPREAD_NS, GAPS_MS[tick] * MS)
        u_arr = t - (rng.random(n) * spread).astype(np.int64)  # not time-sorted
        if self.start is not None:
            u_arr -= self.start[u_cell]
        order = np.argsort(w_cell, kind="stable")
        bc, bs = w_cell[order], w_sub[order]
        cs = np.searchsorted(bc, np.arange(C_ + 1))
        cnt = np.diff(cs)[u_cell]
        pick = cs[u_cell] + (rng.random(n) * np.maximum(cnt, 1)).astype(np.int64)
        u_snd = np.where((rng.random(n) < 0.5) & (cnt > 0), self.conn[bs[np.minimum(pick, max(len(bs) - 1, 0))]], 7).astype(np.uint32)
        return n_cell, u_arr.astype(np.int64), u_snd


class _Reference:
    """The oracle's channels driven like the engine: per tick the interest diff, the updates and tickData, in the order the engine
    applies them (`rings_first`: chd_rings_append before a chd_tick that updates interest; otherwise after chd_update_interest)."""

    def __init__(self, oracle, world, cap, rings_first=False):
        self.o, self.w = oracle, world
        self.chans = oracle.channels(world.C)
        self.groups = None
        if world.start is not None:
            self.groups = [(np.nonzero(world.start == s)[0], int(s)) for s in np.unique(world.start)]
            self.views = [self.chans.view(g) for g, _ in self.groups]
        self.slabs = _Slabs(world.C, cap)
        self.rings_first = rings_first
        self.prev_keys = np.zeros(0, np.int64)
        # what the cases are named for
        self.due = self.multi = self.update_sends = 0
        self.spans, self.multi_staged, self.multi_global = set(), 0, 0
        self.evict_above_max = 0
        self.dists = set()

    def _subscribe(self, w_cell, w_sub, w_iv, t, keys):
        conn = self.w.conn
        gone = np.setdiff1d(self.prev_keys, keys)
        self.chans.unsubscribe(gone & 0xFFFFF, conn[gone >> 20])
        if self.groups is None:
            self.chans.subscribe(w_cell, conn[w_sub], t, w_iv)
        else:  # every channel subscribes in its own time (channel.go:178)
            for g, s in self.groups:
                m = np.isin(w_cell, g)
                self.chans.subscribe(w_cell[m], conn[w_sub[m]], t - s, w_iv[m])
        self.prev_keys = np.sort(keys)

    def _tick_data(self, t, cap):
        if self.groups is None:
            sends, soff = self.chans.tick_data(t, cap)
            return sends, np.repeat(np.arange(self.w.C), np.diff(soff.astype(np.int64)))
        parts, cells = [], []
        for (g, s), v in zip(self.groups, self.views):
            sends, soff = v.tick_data(t - s, cap)
            parts.append(sends)
            cells.append(np.repeat(g, np.diff(soff.astype(np.int64))))
        return np.concatenate(parts), np.concatenate(cells)

    def tick(self, tick, t, want):
        """one tick of the oracle for the sphere_tick result `want` -> dict of what the engine must give"""
        w = self.w
        P = len(want["pair_cell"])
        w_sub = np.repeat(np.arange(w.S), np.diff(want["pair_off"].astype(np.int64)))
        w_cell = want["pair_cell"].astype(np.int64) - S0
        w_iv = _intervals(want["pair_dist"])
        keys = _pair_keys(w_sub, w_cell)
        self.dists |= set(np.unique(want["pair_dist"]).tolist())
        # only the special subscribers watch D
        assert (w_sub[w_cell == w.D] >= w.S - N_SPECIAL).all() and (w_cell == w.D).sum() == N_SPECIAL
        n_cell, u_arr, u_snd = w.updates(tick, w_sub, w_cell)
        if not self.rings_first:
            self._subscribe(w_cell, w_sub, w_iv, t, keys)
        before = self.chans.get_rings()
        ev = self.slabs.append(n_cell, u_arr, before, before["max_interval_ms"])
        self.chans.on_update(np.repeat(np.arange(w.C, dtype=np.uint32), n_cell), u_arr, u_snd)
        if self.rings_first:
            self._subscribe(w_cell, w_sub, w_iv, t, keys)
        rings = self.chans.get_rings()
        np.testing.assert_array_equal(np.diff(rings["off"].astype(np.int64)), self.slabs.e - self.slabs.b)
        # an eviction in D while a kept pair there has a longer interval than D's maxFanOutIntervalMs
        if ev[w.D] and w_iv[w_cell == w.D].max() > rings["max_interval_ms"][w.D]:
            self.evict_above_max += 1
        spans, multi = self.slabs.block_spans(np.sort(w_cell))
        self.spans |= set(spans[multi].tolist())
        self.multi_staged += int((multi & (spans <= FANOUT_STAGE)).sum())
        self.multi_global += int((multi & (spans > FANOUT_STAGE)).sum())
        sends, s_cell = self._tick_data(t, 12 * P + 4096)
        k = sends["conn_id"].astype(np.int64) * (w.C + 1) + s_cell
        self.multi += int((np.unique(k, return_counts=True)[1] > 2).sum())  # pairs with more than FANOUT_SLOTS decisions
        self.due += len(sends)
        self.update_sends += int((sends["kind"] == 1).sum())
        due = _due_table(sends["conn_id"], (s_cell + S0).astype(np.uint32), sends["kind"], sends["n_selected"], sends["first_sel"],
                         sends["last_sel"], sends["sel_hash"], sends["last_message_index"], sends["window_hi"])
        return dict(P=P, w_sub=w_sub, w_cell=w_cell, w_iv=w_iv, upd_off=_csr(n_cell), u_arr=u_arr, u_snd=u_snd, rings=rings, due=due)

    def check_pairs(self, e, r):
        """the engine's pairs (cells, intervals) and every pair's committed fan-out state against the oracle"""
        w = self.w
        pairs = e.get_pairs()
        g_sub = np.repeat(np.arange(w.S), np.diff(pairs["off"].astype(np.int64)))
        g_cell = pairs["channel"].astype(np.int64) - S0
        np.testing.assert_array_equal(np.sort(_pair_keys(g_sub, g_cell)), self.prev_keys)
        go, wo = np.lexsort((g_cell, g_sub)), np.lexsort((r["w_cell"], r["w_sub"]))
        np.testing.assert_array_equal(pairs["interval"][go], r["w_iv"][wo])
        last, had, li, found = self.chans.state(g_cell, w.conn[g_sub])
        assert found.all()
        np.testing.assert_array_equal(pairs["last"], last)
        np.testing.assert_array_equal((pairs["flags"] & 1).astype(bool), had)
        np.testing.assert_array_equal(pairs["last_index"], li)


def _engine(chd, w, cap, graphs=True, n_ent=1, **lim):
    offx, offz = w.g[0], w.g[1]
    e = chd.engine.Engine(chd.engine.grid_cfg(*w.g), max(n_ent, 1), w.S, max_pairs=1 << 21, max_due=1 << 23, max_ring_entries=w.C * cap,
                          max_window_cells=w.S * 48 + 65536, **lim)
    e.enable_graphs(graphs)
    rng = np.random.default_rng(5)
    e.set_entities(offx + rng.random(n_ent) * w.W, offz + rng.random(n_ent) * w.H)  # the fan-out does not depend on entities
    e.set_subscribers(w.conn)
    e.build()
    if w.start is not None:
        start = np.ascontiguousarray(w.start)
        assert e.L.chd_set_channel_start_times(e.h, chd.capi.ptr(start)) == chd.capi.OK
    e.rings_init(cap)
    return e


def _due_from(conn, d):
    return _due_table(conn[d["sub"]], d["channel_id"], d["kind"], d["n_selected"], d["first_sel"], d["last_sel"], d["sel_hash"],
                      d["last_message_index"], d["window_hi"])


@pytest.mark.parametrize("grid,cap,starts", CASES)
def test_rings_scale_parity(chd, oracle, grid, cap, starts):
    """chd_update_interest, chd_rings_append, chd_fanout_tick for 8 irregular ticks: every tick the rings (offsets, every entry,
    msgIndex), the due list as a set, every pair's committed state and a clean overflow mask equal the oracle's."""
    stage = cap == 620
    w = _World(oracle, grid, 4000 + cap + 7 * starts + ord(grid), stage=stage, starts=starts)
    ref = _Reference(oracle, w, cap)
    e = _engine(chd, w, cap)
    for tick in range(N_TICKS):
        t, cx, cz, rad = w.next_tick(tick)
        want = oracle.sphere_pairs(w.og, np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]), cx, cz, rad)
        assert (want["status"] == 0).all()
        batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(cx, cz, rad))
        e.update_interest(batch, t)
        s = e.summary()
        r = ref.tick(tick, t, want)
        assert s.n_pairs == r["P"] and s.overflow == 0
        e.rings_append(r["upd_off"], r["u_arr"], r["u_snd"])
        _assert_rings(e.get_rings(), r["rings"])
        e.fanout_tick(t)
        s = e.summary()
        assert s.overflow == 0 and s.n_due == len(r["due"])
        np.testing.assert_array_equal(_due_from(w.conn, e.get_due(s.n_due)), r["due"])
        ref.check_pairs(e, r)
    e.close()
    # every case runs the paths it is named for
    sl = ref.slabs
    assert ref.dists >= {0, 1, 2}
    assert ref.due > 100_000 and ref.multi > 1000 and ref.update_sends > 1000
    assert ref.multi_global > 0
    assert sl.drops.sum() == 0
    if stage:
        assert FANOUT_STAGE in ref.spans and FANOUT_STAGE + 1 in ref.spans and ref.multi_staged > 0
    else:
        assert (sl.evictions > 0).sum() >= 10 and sl.slides.sum() > 0 and ref.evict_above_max > 0
        if cap == 513 and grid != "e":
            assert ref.multi_staged > 0


def _script(chd, oracle, w, cap, rings_first):
    """the oracle's side of N_TICKS ticks -> per tick (t, batch arrays, reference results), and the reference"""
    ref = _Reference(oracle, w, cap, rings_first=rings_first)
    out = []
    for tick in range(N_TICKS):
        t, cx, cz, rad = w.next_tick(tick)
        want = oracle.sphere_pairs(w.og, np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]), cx, cz, rad)
        out.append((t, (cx, cz, rad), ref.tick(tick, t, want)))
    return out, ref


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "nographs"])
def test_rings_under_the_two_stream_tick(chd, oracle, graphs):
    """chd_rings_append, then chd_tick(TICK_ALL) (interest update and fan-out on the second stream, beside the build and the
    copy): rings, due lists and pair state equal the oracle's every tick."""
    w = _World(oracle, "b", 77, n_sub=40_000)
    cap = 1024
    script, ref = _script(chd, oracle, w, cap, rings_first=True)
    e = _engine(chd, w, cap, graphs=graphs, n_ent=2000, max_visible=1 << 24)
    ref_final = None
    for tick, (t, q, r) in enumerate(script):
        e.rings_append(r["upd_off"], r["u_arr"], r["u_snd"])
        batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=q)
        s = e.tick(batch, t, chd.capi.TICK_ALL)
        assert s.overflow == 0 and s.n_pairs == r["P"] and s.n_due == len(r["due"])
        np.testing.assert_array_equal(_due_from(w.conn, e.get_due(s.n_due)), r["due"])
        _assert_rings(e.get_rings(), r["rings"])
        ref_final = r
    ref.check_pairs(e, ref_final)
    assert (ref.slabs.evictions > 0).sum() >= 10 and ref.slabs.slides.sum() > 0
    e.close()


def test_rings_in_the_pipelined_loop(chd, oracle):
    """The pipelined loop: tick k+1's chd_rings_append is enqueued while tick k's copy kernel runs and before its results are
    waited for (chd_fetch_results_async / chd_fetch_wait, two result sets).  Due lists of every tick and the final pair state
    equal the oracle's."""
    torch = chd.torch
    w = _World(oracle, "b", 78, n_sub=40_000)
    cap = 1024
    script, ref = _script(chd, oracle, w, cap, rings_first=True)
    e = _engine(chd, w, cap, n_ent=2000, max_visible=1 << 24)
    due_cap = 1 << 22
    sets = []
    for _ in range(2):
        d = torch.zeros(due_cap * 12, dtype=torch.int32).pin_memory()
        hdr = torch.zeros(64, dtype=torch.int32).pin_memory()
        rb = chd.capi.ResultBuffers()
        rb.due, rb.due_cap = chd.capi.ptr(d), due_cap
        sets.append((rb, d, hdr))
    s = chd.capi.TickSummary()
    keep = []

    def check(i):
        rb, d, hdr = sets[i % 2]
        r = script[i][2]
        assert s.overflow == 0 and s.n_due == len(r["due"]), i
        got = d.numpy().view(chd.capi.DUE_DTYPE)[:s.n_due]
        np.testing.assert_array_equal(_due_from(w.conn, got), r["due"], err_msg=str(i))

    for i, (t, q, r) in enumerate(script):
        e.rings_append(r["upd_off"], r["u_arr"], r["u_snd"])
        batch, kb = chd.engine.make_batch(w.S, sub=None, sphere=q)
        keep.append((batch, kb))
        e.tick(batch, t, chd.capi.TICK_ALL, want_summary=False)
        rb, d, hdr = sets[i % 2]
        e._ck(e.L.chd_fetch_results_async(e.h, C.byref(rb), chd.capi.ptr(hdr)))
        if i:
            e._ck(e.L.chd_fetch_wait(e.h, C.byref(s)))
            check(i - 1)
    e._ck(e.L.chd_fetch_wait(e.h, C.byref(s)))
    check(len(script) - 1)
    ref.check_pairs(e, script[-1][2])
    _assert_rings(e.get_rings(), script[-1][2]["rings"])
    e.close()


def _small(chd, oracle, cap, n_sub=2000, seed=9, **lim):
    """the 300-cell grid with n_sub subscribers (none near D) and device-owned rings of `cap` entries per cell"""
    w = _World(oracle, "b", seed, n_sub=n_sub, n_hot=0)
    w.hot[:] = False
    e = _engine(chd, w, cap, **lim)
    return w, e


def _interest(chd, oracle, w, e, ref, tick):
    t, cx, cz, rad = w.next_tick(tick)
    want = oracle.sphere_pairs(w.og, np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]), cx, cz, rad)
    batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(cx, cz, rad))
    e.update_interest(batch, t)
    e.summary()
    w_sub = np.repeat(np.arange(w.S), np.diff(want["pair_off"].astype(np.int64)))
    w_cell = want["pair_cell"].astype(np.int64) - S0
    keys = _pair_keys(w_sub, w_cell)
    ref._subscribe(w_cell, w_sub, _intervals(want["pair_dist"]), t, keys)
    return t, dict(w_sub=w_sub, w_cell=w_cell, w_iv=_intervals(want["pair_dist"]), batch=(batch, keep), q=(cx, cz, rad))


def _due_by_cell(ref, t, skip=()):
    sends, s_cell = ref._tick_data(t, 1 << 22)
    m = ~np.isin(s_cell, list(skip))
    sends, s_cell = sends[m], s_cell[m]
    return _due_table(sends["conn_id"], (s_cell + S0).astype(np.uint32), sends["kind"], sends["n_selected"], sends["first_sel"],
                      sends["last_sel"], sends["sel_hash"], sends["last_message_index"], sends["window_hi"])


def test_full_slab_drops_its_oldest_entry(chd, oracle):
    """A cell whose 513-entry slab fills with entries none of which may be evicted (equal arrivals): CHD_OVF_RING, chd_summary
    returns CHD_ERR_CAPACITY, the ring keeps the newest 513 entries and msgIndex counts every update; every other cell, and its
    fan-out, still equals the oracle, and the next tick's mask is clean."""
    capi = chd.capi
    cap = 513
    w, e = _small(chd, oracle, cap)
    ref = _Reference(oracle, w, cap)
    rng = np.random.default_rng(3)
    t, p = _interest(chd, oracle, w, e, ref, 0)
    X = int(np.bincount(p["w_cell"], minlength=w.C).argmax())  # the busiest cell
    n_cell = rng.integers(0, 9, w.C)
    n_cell[X] = 600
    u_cell = np.repeat(np.arange(w.C), n_cell)
    u_arr = np.where(u_cell == X, t, t - rng.integers(0, 100 * MS, len(u_cell))).astype(np.int64)
    u_snd = np.full(len(u_cell), 7, np.uint32)
    ref.chans.on_update(u_cell.astype(np.uint32), u_arr, u_snd)
    e.rings_append(_csr(n_cell), u_arr, u_snd)
    e.fanout_tick(t)
    s = capi.TickSummary()
    assert e.L.chd_summary(e.h, C.byref(s)) == capi.ERR_CAPACITY
    assert s.overflow == capi.OVF_RING
    got, want = e.get_rings(), ref.chans.get_rings()
    _assert_rings(got, want, skip=[X])
    g0, w0 = int(got["off"][X]), int(want["off"][X])
    assert int(got["off"][X + 1]) - g0 == cap and int(want["off"][X + 1]) - w0 == 600
    for k in ("arrival", "sender", "index"):
        np.testing.assert_array_equal(got[k][g0:g0 + cap], want[k][w0 + 600 - cap:w0 + 600])
    assert got["msg_index"][X] == 600
    # the fan-out of every other cell
    due = _due_from(w.conn, e.get_due(s.n_due))
    due = due[due["channel"] != S0 + X]
    np.testing.assert_array_equal(due, _due_by_cell(ref, t, skip=[X]))
    # next tick: a few updates elsewhere, a clean mask
    t, p = _interest(chd, oracle, w, e, ref, 1)
    n_cell = rng.integers(0, 9, w.C)
    n_cell[X] = 0
    u_cell = np.repeat(np.arange(w.C), n_cell)
    u_arr = (t - rng.integers(0, 100 * MS, len(u_cell))).astype(np.int64)
    u_snd = np.full(len(u_cell), 7, np.uint32)
    ref.chans.on_update(u_cell.astype(np.uint32), u_arr, u_snd)
    e.rings_append(_csr(n_cell), u_arr, u_snd)
    e.fanout_tick(t)
    assert e.L.chd_summary(e.h, C.byref(s)) == capi.OK and s.overflow == 0
    _assert_rings(e.get_rings(), ref.chans.get_rings(), skip=[X])
    due = _due_from(w.conn, e.get_due(s.n_due))
    np.testing.assert_array_equal(due[due["channel"] != S0 + X], _due_by_cell(ref, t, skip=[X]))
    e.close()


def test_ring_argument_edges(chd, oracle):
    """Capacity limits of chd_rings_init, an empty append, two appends in one tick against one concatenated append, an append that
    grows the upload buffers, a CSR whose last offset overshoots n_updates, and chd_assemble_payloads on device-owned rings."""
    capi = chd.capi
    p = capi.ptr
    rng = np.random.default_rng(11)
    w = _World(oracle, "b", 12, n_sub=2000, n_hot=0)
    C_ = w.C
    e = chd.engine.Engine(chd.engine.grid_cfg(*w.g), 16, w.S, max_ring_entries=C_ * 1024)
    assert _status(lambda: e.rings_init(512)) == capi.ERR_INVALID
    assert _status(lambda: e.rings_init(1025)) == capi.ERR_CAPACITY
    e.rings_init(513)
    e.rings_init(1024)  # cells x cap == max_ring_entries
    e_one_less = chd.engine.Engine(chd.engine.grid_cfg(*w.g), 16, w.S, max_ring_entries=C_ * 1024 - 1)
    assert _status(lambda: e_one_less.rings_init(1024)) == capi.ERR_CAPACITY
    e_one_less.rings_init(1023)
    e_one_less.close()
    e2 = chd.engine.Engine(chd.engine.grid_cfg(*w.g), 16, w.S, max_ring_entries=C_ * 1024)
    e2.rings_init(1024)
    chans = oracle.channels(C_)

    def updates(lo, hi, t):
        n_cell = rng.integers(lo, hi, C_)
        u_cell = np.repeat(np.arange(C_), n_cell)
        return n_cell, (t - rng.integers(0, 200 * MS, len(u_cell))).astype(np.int64), rng.integers(1, 50, len(u_cell)).astype(np.uint32)

    # an append without updates changes nothing
    zero = np.zeros(C_ + 1, np.uint32)
    assert e.L.chd_rings_append(e.h, p(zero), 0, None, None) == capi.OK
    assert int(e.get_rings()["off"][-1]) == 0
    # two appends in one tick == the same updates concatenated per cell in one append (and == the oracle)
    n1, a1, s1 = updates(0, 30, 1000 * MS)
    n2, a2, s2 = updates(0, 30, 1000 * MS)
    for n_, a_, s_ in ((n1, a1, s1), (n2, a2, s2)):
        e.rings_append(_csr(n_), a_, s_)
        chans.on_update(np.repeat(np.arange(C_, dtype=np.uint32), n_), a_, s_)
    o1, o2 = _csr(n1).astype(np.int64), _csr(n2).astype(np.int64)
    cat = [np.concatenate([x[o1[c]:o1[c + 1]], y[o2[c]:o2[c + 1]]]) for c in range(C_) for x, y in [(a1, a2)]]
    cat_s = [np.concatenate([x[o1[c]:o1[c + 1]], y[o2[c]:o2[c + 1]]]) for c in range(C_) for x, y in [(s1, s2)]]
    e2.rings_append(_csr(n1 + n2), np.concatenate(cat), np.concatenate(cat_s))
    got = e.get_rings()
    _assert_rings(got, chans.get_rings())
    _assert_rings(e2.get_rings(), got)
    # an append larger than the upload buffers (they grow), with floods past 512 in every cell
    n3, a3, s3 = updates(600, 700, 1300 * MS)
    assert n3.sum() > 150_000
    e.rings_append(_csr(n3), a3, s3)
    chans.on_update(np.repeat(np.arange(C_, dtype=np.uint32), n3), a3, s3)
    _assert_rings(e.get_rings(), chans.get_rings())
    # a CSR that claims 3 entries more than n_updates (still inside the grown upload buffers, which hold stale updates there):
    # only the first n_updates are appended
    n4, a4, s4 = updates(0, 9, 1500 * MS)
    off4 = _csr(n4)
    n_upd = int(off4[-1])
    off4[-1] += 3
    a4p, s4p = np.concatenate([a4, np.full(3, 1500 * MS, np.int64)]), np.concatenate([s4, np.full(3, 99, np.uint32)])
    e.rings_append(off4, a4p, s4p, n=n_upd)
    chans.on_update(np.repeat(np.arange(C_, dtype=np.uint32), n4), a4, s4)
    _assert_rings(e.get_rings(), chans.get_rings())
    # chd_assemble_payloads indexes payload bytes by ring position: refused on device-owned rings
    e.set_subscribers(w.conn)
    e.set_entities(np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]))
    e.build()
    t, cx, cz, rad = w.next_tick(0)
    batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(cx, cz, rad))
    e.update_interest(batch, 1000 * MS)
    e.fanout_tick(1600 * MS)
    s = e.summary()
    assert s.n_due > 0
    eoff, foff = np.zeros(1, np.uint64), np.zeros(C_ + 1, np.uint64)
    assert e.L.chd_set_payload_bytes(e.h, p(eoff), 0, None, p(foff), None, b"type.googleapis.com/x", 0) == capi.OK
    ncls, blen = C.c_uint32(0), C.c_uint64(0)
    cls_off, blob = np.zeros(s.n_due + 1, np.uint64), np.zeros(1 << 16, np.uint8)
    assert e.L.chd_assemble_payloads(e.h, C.byref(ncls), p(cls_off), s.n_due + 1, p(blob), blob.size, C.byref(blen)) == capi.ERR_STATE
    e.close()
    e2.close()


def test_ring_inputs_are_refused_while_a_begun_interest_chain_reads_them(chd, oracle):
    """chd_begin_interest forks the interest update and the fan-out onto the engine's second stream, which reads the rings, the
    channel start times and the per-channel maxFanOutIntervalMs.  Until chd_tick joins it, chd_rings_append, chd_rings_init and
    chd_set_channel_start_times return CHD_ERR_STATE and change nothing; chd_set_rings does when the begun chain includes the
    fan-out, and is accepted without it."""
    capi = chd.capi
    p = capi.ptr
    cap = 1024
    w, e = _small(chd, oracle, cap, seed=21)
    ref = _Reference(oracle, w, cap)
    rng = np.random.default_rng(22)
    C_ = w.C
    # tick 0 in full
    t, pi = _interest(chd, oracle, w, e, ref, 0)
    n0 = rng.integers(0, 9, C_)
    a0 = (t - rng.integers(0, 100 * MS, n0.sum())).astype(np.int64)
    s0 = np.full(n0.sum(), 7, np.uint32)
    e.rings_append(_csr(n0), a0, s0)
    ref.chans.on_update(np.repeat(np.arange(C_, dtype=np.uint32), n0), a0, s0)
    e.fanout_tick(t)
    s = e.summary()
    np.testing.assert_array_equal(_due_from(w.conn, e.get_due(s.n_due)), _due_by_cell(ref, t))
    # tick 1: its updates, then chd_begin_interest with the fan-out; every ring input is refused until chd_tick
    t1, cx, cz, rad = w.next_tick(1)
    n1 = rng.integers(0, 9, C_)
    a1 = (t1 - rng.integers(0, 100 * MS, n1.sum())).astype(np.int64)
    s1 = np.full(n1.sum(), 7, np.uint32)
    e.rings_append(_csr(n1), a1, s1)
    ref.chans.on_update(np.repeat(np.arange(C_, dtype=np.uint32), n1), a1, s1)
    want = oracle.sphere_pairs(w.og, np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]), cx, cz, rad)
    w_sub = np.repeat(np.arange(w.S), np.diff(want["pair_off"].astype(np.int64)))
    w_cell = want["pair_cell"].astype(np.int64) - S0
    ref._subscribe(w_cell, w_sub, _intervals(want["pair_dist"]), t1, _pair_keys(w_sub, w_cell))
    batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(cx, cz, rad))
    e.begin_interest(batch, t1, with_fanout=True)
    bad = rng.integers(1, 5, C_)
    bad_a = np.full(bad.sum(), t1, np.int64)
    bad_s = np.full(bad.sum(), 8, np.uint32)
    assert _status(lambda: e.rings_append(_csr(bad), bad_a, bad_s)) == capi.ERR_STATE
    assert _status(lambda: e.rings_init(cap)) == capi.ERR_STATE
    start = np.full(C_, 5 * MS, np.int64)
    assert e.L.chd_set_channel_start_times(e.h, p(start)) == capi.ERR_STATE
    s = e.tick(None, t1, capi.TICK_ALL)
    assert s.overflow == 0
    _assert_rings(e.get_rings(), ref.chans.get_rings())
    np.testing.assert_array_equal(_due_from(w.conn, e.get_due(s.n_due)), _due_by_cell(ref, t1))
    e.close()

    # host-owned rings: chd_set_rings is refused while a begun chain includes the fan-out, accepted while it does not
    w2 = _World(oracle, "b", 23, n_sub=2000, n_hot=0)
    e = chd.engine.Engine(chd.engine.grid_cfg(*w2.g), 16, w2.S, max_ring_entries=C_ * 64)
    e.set_entities(np.array([w2.g[0] + 1.0]), np.array([w2.g[1] + 1.0]))
    e.set_subscribers(w2.conn)
    e.build()
    ref = _Reference(oracle, w2, 64)
    for tick, with_fanout in ((0, True), (1, True), (2, False), (3, False)):
        t, cx, cz, rad = w2.next_tick(tick)
        want = oracle.sphere_pairs(w2.og, np.array([w2.g[0] + 1.0]), np.array([w2.g[1] + 1.0]), cx, cz, rad)
        w_sub = np.repeat(np.arange(w2.S), np.diff(want["pair_off"].astype(np.int64)))
        w_cell = want["pair_cell"].astype(np.int64) - S0
        ref._subscribe(w_cell, w_sub, _intervals(want["pair_dist"]), t, _pair_keys(w_sub, w_cell))
        # the oracle's channels take this tick's updates; the engine gets their whole buffers as the ring snapshot
        n_ = rng.integers(0, 9, C_)
        a_ = (t - rng.integers(0, 100 * MS, n_.sum())).astype(np.int64)
        s_ = np.full(n_.sum(), 7, np.uint32)
        ref.chans.on_update(np.repeat(np.arange(C_, dtype=np.uint32), n_), a_, s_)
        r = ref.chans.get_rings()
        ring = (r["off"].astype(np.uint32), r["arrival"], r["sender"], r["index"], r["msg_index"])
        batch, keep = chd.engine.make_batch(w2.S, sub=None, sphere=(cx, cz, rad))
        if with_fanout:
            e.set_rings(*ring)
            e.begin_interest(batch, t, with_fanout=True)
            # another snapshot (every entry from connection 8, arriving at t) is refused: the begun fan-out reads the rings
            ro, ri, rc = (np.ascontiguousarray(x) for x in (ring[0], ring[3], ring[4]))
            ra, rs = np.full(len(ri), t, np.int64), np.full(len(ri), 8, np.uint32)
            assert e.L.chd_set_rings(e.h, p(ro), int(ro[-1]), p(ra), p(rs), p(ri), p(rc)) == capi.ERR_STATE
        else:
            e.begin_interest(batch, t, with_fanout=False)
            e.set_rings(*ring)  # accepted: the begun chain does not read the rings, chd_tick runs the fan-out after it
        s = e.tick(None, t, capi.TICK_ALL)
        assert s.overflow == 0 and (s.n_due > 0 or tick == 0)
        np.testing.assert_array_equal(_due_from(w2.conn, e.get_due(s.n_due)), _due_by_cell(ref, t))
    e.close()
