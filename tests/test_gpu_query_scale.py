"""QueryChannelIds (spatial.go:182-317) and handleUpdateSpatialInterest for every AOI kind against the oracle at the sizes where
query_kernel / interest_fill_kernel (chd_query.cuh, chd_interest.cuh) do what small tests never reach: windows of 1000+ cells,
side lists of 64+ spots that interleave with the window's cell ids, batches of thousands of 128-query blocks, and a window scratch
that runs out (CHD_OVF_WINDOW fails queries one by one, in an order that depends on block scheduling).  The queries come from
tests/_queries.py (all 16 kind masks, cell-edge centres and radii, cones at the world edge, every error path); each query's
window size comes from a numpy restatement of query_bbox.
Run on an H100:  python -m pytest tests/test_gpu_query_scale.py -m gpu
"""
import concurrent.futures as cf
import ctypes as C
import os

import numpy as np
import pytest

from tests import _queries as Q

pytestmark = pytest.mark.gpu

S0 = 65536
MS = 1_000_000

# (grid, number of queries, reach of the long shapes in cells, what the grid must produce: windows of 1000+ cells, side lists of
# 64+ spots, side cells interleaved with window cells)
GRIDS = {
    "benchmark_15x15": ((-15000, -15000, 2000, 2000, 15, 15), 100_000, 20.0, (False, True, True)),
    "256x256": ((-12800, -12800, 100, 100, 256, 256), 1 << 19, 20.0, (True, True, True)),
    "600x400_odd": ((-12.5, 3.25, 7.3, 11.9, 600, 400), 100_000, 20.0, (True, True, True)),
    "4096x3": ((0, 0, 50, 50, 4096, 3), 100_000, 200.0, (True, True, True)),
    "3x4096": ((0, 0, 50, 50, 3, 4096), 100_000, 200.0, (True, True, True)),
}


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
    ns.capi, ns.engine = capi, engine
    return ns


def _threads():
    return os.cpu_count() or 1


def _coverage(grid, q, st, off, ids):
    """-> (largest window of an answered query, largest side list, side cells whose id lies between two window cells of the same
    answer).  Side list = the distinct in-world spot cells outside the window (the kernel's per-query list)."""
    offx, offz, w, h, cols, rows = grid
    gx0, gy0, bw, bh = Q.query_windows(grid, q)
    ok = st == 0
    wn = bw * bh
    # side lists
    soff, _, sx, sz, _ = q["spots"]
    owner = np.repeat(np.arange(q["n"]), np.diff(soff.astype(np.int64)))
    v, gx, gy = Q.grid_coord(grid, sx, sz)
    inside = (gx - gx0[owner] >= 0) & (gx - gx0[owner] < bw[owner]) & (gy - gy0[owner] >= 0) & (gy - gy0[owner] < bh[owner])
    side = v & ~inside & ok[owner] & ((q["kind"][owner] & Q.AOI_SPOTS) != 0)
    keys = np.unique(owner[side].astype(np.int64) * (cols * rows) + gx[side] + gy[side] * cols)
    side_len = np.bincount(keys // (cols * rows), minlength=q["n"])
    # interleaving, on the answers themselves
    rown = np.repeat(np.arange(q["n"]), np.diff(off.astype(np.int64)))
    c = ids.astype(np.int64) - S0
    cx_, cy_ = c % cols, c // cols
    inw = (cx_ - gx0[rown] >= 0) & (cx_ - gx0[rown] < bw[rown]) & (cy_ - gy0[rown] >= 0) & (cy_ - gy0[rown] < bh[rown])
    lo = np.full(q["n"], np.iinfo(np.int64).max)
    hi = np.full(q["n"], -1)
    np.minimum.at(lo, rown[inw], c[inw])
    np.maximum.at(hi, rown[inw], c[inw])
    between = (~inw) & (c > lo[rown]) & (c < hi[rown])
    return int(wn[ok].max(initial=0)), int(side_len.max(initial=0)), int(between.sum())


@pytest.mark.parametrize("name", list(GRIDS))
def test_stateless_queries_at_scale(chd, oracle, name):
    """chd_query_channel_ids on 100 K+ queries of every kind against orc_query_batch: statuses exact, the CSR equal array for
    array.  The window scratch is exactly the restated requirement (the call succeeds); one cell less fails the batch and
    reports the requirement."""
    from tests._oracle import make_grid

    grid, n, long_cells, (want_big, want_side, want_between) = GRIDS[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    q = Q.make_queries(rng, grid, n, long_cells=long_cells)
    gx0, gy0, bw, bh = Q.query_windows(grid, q)
    need = int((bw * bh).sum())
    st, off, ids, dist = oracle.query_batch(make_grid(*grid), n, n_threads=_threads(), **Q.batch_kwargs(q))
    total = int(off[-1])
    big, side, between = _coverage(grid, q, st, off, ids)
    assert (not want_big or big >= 1000) and (not want_side or side >= 64) and (not want_between or between >= 1), (big, side, between)
    assert (n + 127) // 128 >= (4096 if n >= 1 << 19 else 700)  # thousands of 128-query blocks reserve window scratch
    assert set(q["kind"].tolist()) == set(range(16)) and {0, 1, 2, 5}.issubset(set(st.tolist()))
    n_spots = int(q["spots"][0][-1])
    lim = dict(max_queries=n, max_spots=n_spots + 1, max_pairs=total + 1024)
    cfg = chd.engine.grid_cfg(*grid)
    e = chd.engine.Engine(cfg, 16, n, max_window_cells=need, **lim)
    batch, keep = chd.engine.make_batch(n, **Q.batch_kwargs(q))
    gst, goff, gids, gdist = e.query_channel_ids(batch, cap=total + 16)
    np.testing.assert_array_equal(gst, st)
    np.testing.assert_array_equal(goff.astype(np.uint64), off)
    np.testing.assert_array_equal(gids, ids)
    np.testing.assert_array_equal(gdist, dist)
    e.close()
    short = chd.engine.Engine(cfg, 16, n, max_window_cells=need - 1, **lim)
    with pytest.raises(chd.capi.ChdError) as ei:
        short.query_channel_ids(batch, cap=total + 16)
    assert ei.value.status == chd.capi.ERR_CAPACITY and f"need {need} cells" in str(ei.value)
    short.close()


# ---------------------------------------------------------------- the interest update, six ticks of 100 K subscribers

WORLD = (-12800, -12800, 100, 100, 256, 256)
S, N, TICKS = 100_000, 400_000, 6
DELAY_MS, DEFAULT_MS = 7, 30


def _world(seed=2024):
    """Entities (2 % outside the world) and per tick: the positions, the queried slots (a random ~70 % in permuted order) and
    their queries, with centres that move and kinds that change."""
    offx, offz, w, h, cols, rows = WORLD
    rng = np.random.default_rng(seed)
    ex, ez = offx + rng.uniform(0, 1, N) * w * cols, offz + rng.uniform(0, 1, N) * h * rows
    out = rng.random(N) < 0.02
    ex[out] = offx - rng.uniform(1, 500, out.sum())
    cx, cz = offx + rng.uniform(0, 1, S) * w * cols, offz + rng.uniform(0, 1, S) * h * rows
    kind = rng.integers(0, 16, S).astype(np.uint8)
    ticks = []
    for t in range(TICKS):
        ex = ex + rng.uniform(-60, 60, N)
        ez = ez + rng.uniform(-60, 60, N)
        cx = np.clip(cx + rng.uniform(-150, 150, S), offx, offx + w * cols - 1)
        cz = np.clip(cz + rng.uniform(-150, 150, S), offz, offz + h * rows - 1)
        ch = rng.random(S) < 0.15
        kind[ch] = rng.integers(0, 16, ch.sum())
        slots = rng.permutation(np.nonzero(rng.random(S) < 0.7)[0]).astype(np.uint32)
        q = Q.make_queries(rng, WORLD, len(slots), cx=cx[slots], cz=cz[slots], kind=kind[slots], p_err=0.005, long_cells=20.0,
                           max_spots=120)
        gx0, gy0, bw, bh = Q.query_windows(WORLD, q)
        ticks.append(dict(t=(t + 1) * 100 * MS, ex=ex.copy(), ez=ez.copy(), slots=slots, q=q, wn=bw * bh))
    return ticks


class Model:
    """The engine's pairs as the oracle says they must be: per slot a run of (channel, dist) ascending, with fan-out state."""

    def __init__(self):
        self.off = np.zeros(S + 1, np.int64)
        self.f = {k: np.zeros(0, dt) for k, dt in (("channel", np.uint32), ("dist", np.uint32), ("flags", np.uint8), ("last", np.int64),
                                                    ("last_index", np.uint64))}
        self.box_run = np.zeros(S, bool)  # the slot's current run came from a query with a box

    def keys(self, off, channel):
        return np.repeat(np.arange(S, dtype=np.int64), np.diff(off)) << 32 | channel.astype(np.int64)

    def update(self, slots, ok, qoff, qch, qdist, now_ns, kinds):
        """slot slots[k] takes query k's answer where ok[k]; -> (new keys, unsub keys, n_kept)"""
        qoff = qoff.astype(np.int64)
        P = len(self.f["channel"])
        lens, src = np.diff(self.off), self.off[:-1].copy()
        s_ok = slots[ok].astype(np.int64)
        lens[s_ok] = np.diff(qoff)[ok]
        src[s_ok] = qoff[:-1][ok] + P
        off = np.concatenate([[0], np.cumsum(lens)])
        idx = np.repeat(src - off[:-1], lens) + np.arange(off[-1])
        from_q = idx >= P
        ch = np.concatenate([self.f["channel"], qch.astype(np.uint32)])[idx]
        dist = np.concatenate([self.f["dist"], qdist.astype(np.uint32)])[idx]
        old_keys = self.keys(self.off, self.f["channel"])
        new_keys = self.keys(off, ch)
        pos = np.minimum(np.searchsorted(old_keys, new_keys), max(P - 1, 0))
        found = (P > 0) & (old_keys[pos] == new_keys) if P else np.zeros(len(new_keys), bool)
        take = np.where(found, pos, 0)
        g = {}
        g["flags"] = np.where(found, self.f["flags"][take] & ~np.uint8(2) if P else 0, 2 | 4).astype(np.uint8)
        g["last"] = np.where(found, self.f["last"][take] if P else 0, now_ns + DELAY_MS * MS).astype(np.int64)
        g["last_index"] = np.where(found, self.f["last_index"][take] if P else 0, 0).astype(np.uint64)
        assert (found | from_q).all()  # an untouched run is found in the old state
        queried = np.zeros(S, bool)
        queried[s_ok] = True
        new = new_keys[from_q & ~found]
        old_slot = np.repeat(np.arange(S), np.diff(self.off))
        gone = old_keys[queried[old_slot] & ~np.isin(old_keys, new_keys)]
        n_kept = int((from_q & found).sum())
        self.off = off
        self.f = dict(channel=ch, dist=dist, **g)
        self.box_run[s_ok] = (kinds[ok] & Q.AOI_BOX) != 0
        return new, gone, n_kept


def _check_pairs(oracle, pairs, m):
    np.testing.assert_array_equal(pairs["off"].astype(np.int64), m.off)
    for k in ("channel", "dist", "flags", "last", "last_index"):
        np.testing.assert_array_equal(pairs[k], m.f[k], err_msg=k)
    u = np.unique(m.f["dist"])
    lut = np.array([oracle.damping(int(d), DEFAULT_MS) for d in u], np.uint32)
    np.testing.assert_array_equal(pairs["interval"], lut[np.searchsorted(u, m.f["dist"])])
    return int(len(u))


def _canon(a, b):
    return np.sort(a.astype(np.int64) << 32 | b.astype(np.int64))


def _engine(chd, window_cells):
    e = chd.engine.Engine(chd.engine.grid_cfg(*WORLD), N, S, max_queries=S, max_spots=1 << 23, max_pairs=1 << 25,
                          max_window_cells=int(window_cells), max_visible=1 << 27, max_due=1 << 23, default_fanout_interval_ms=DEFAULT_MS,
                          default_fanout_delay_ms=DELAY_MS)
    e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
    cells = WORLD[4] * WORLD[5]
    e.set_rings(np.zeros(cells + 1, np.uint32), np.zeros(0, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint64))
    return e


def _fanout_between_ticks(e, m, t):
    """A fan-out pass with empty rings 40 ms after the update: due pairs (intervals 20 and 30 ms) take their first FULL fan-out,
    so kept pairs carry a fan-out state of their own into the next update.  The committed state becomes the model's."""
    e.fanout_tick(t + 40 * MS)
    s = e.summary()
    p = e.get_pairs(s.n_pairs)
    np.testing.assert_array_equal(p["channel"], m.f["channel"])
    np.testing.assert_array_equal(p["dist"], m.f["dist"])
    for k in ("flags", "last", "last_index"):
        m.f[k] = p[k].copy()
    return s.n_due


_FINAL = {}


def _run_stateful(chd, oracle, use_graphs):
    from tests._oracle import make_grid

    og = make_grid(*WORLD)
    ticks = _world()
    e = _engine(chd, max(int(tk["wn"].sum()) for tk in ticks) + 1)
    e.enable_graphs(use_graphs)
    m = Model()
    cells = WORLD[4] * WORLD[5]
    n_due = n_kept_total = n_fail = 0
    for tk in ticks:
        q, slots, t = tk["q"], tk["slots"], tk["t"]
        e.set_entities(tk["ex"], tk["ez"])
        batch, keep = chd.engine.make_batch(q["n"], sub=slots, **Q.batch_kwargs(q))
        s = e.tick(batch, t, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT)
        st, qoff, qch, qdist = oracle.query_batch(og, q["n"], n_threads=_threads(), **Q.batch_kwargs(q))
        assert s.overflow == 0 and s.required_window_cells == int(tk["wn"].sum())
        np.testing.assert_array_equal(e.get_query_status(q["n"]), st)
        assert s.n_query_errors == int((st != 0).sum())
        n_fail += int((st != 0).sum())
        new, gone, n_kept = m.update(slots, st == 0, qoff, qch, qdist, t, q["kind"])
        assert (s.n_sub_new, s.n_unsub, s.n_kept) == (len(new), len(gone), n_kept)
        assert s.n_pairs == len(m.f["channel"])
        pairs = e.get_pairs(s.n_pairs)
        _check_pairs(oracle, pairs, m)
        (ns, nc), (us, uc) = e.get_diff(s.n_sub_new, s.n_unsub)
        np.testing.assert_array_equal(_canon(ns, nc), np.sort(new))
        np.testing.assert_array_equal(_canon(us, uc), np.sort(gone))
        # visible lists: the pairs expanded over a stable sort of the oracle's cell ids
        ids = oracle.cell_of(og, tk["ex"], tk["ez"])
        valid = np.nonzero(ids)[0]
        order = valid[np.argsort(ids[valid], kind="stable")].astype(np.uint32)
        cs = np.concatenate([[0], np.cumsum(np.bincount(ids[valid] - S0, minlength=cells))])
        pc = m.f["channel"].astype(np.int64) - S0
        lens = cs[pc + 1] - cs[pc]
        pvo = np.concatenate([[0], np.cumsum(lens)])
        want_vis = order[np.repeat(cs[pc] - pvo[:-1], lens) + np.arange(pvo[-1])]
        want_voff = pvo[m.off]
        voff, vis = e.get_visible()
        np.testing.assert_array_equal(voff.astype(np.int64), want_voff)
        np.testing.assert_array_equal(vis, want_vis)
        assert s.n_visible == len(want_vis) and s.n_entities_in_world == len(valid)
        n_kept_total += n_kept
        n_due += _fanout_between_ticks(e, m, t)
    # what this world is there for
    assert 0.01 * sum(tk["q"]["n"] for tk in ticks) < n_fail < 0.04 * sum(tk["q"]["n"] for tk in ticks)
    assert n_kept_total > 100_000 and n_due > 100_000
    assert ((m.f["flags"] & 1) != 0).sum() > 10_000  # kept pairs carry a first fan-out into the updates
    if use_graphs:
        assert e.graph_launch_count() > 0
    else:
        assert e.graph_launch_count() == 0
    return e, m


@pytest.mark.parametrize("use_graphs", [True, False], ids=["graphs", "direct"])
def test_interest_update_at_scale(chd, oracle, use_graphs):
    """chd_tick(TICK_BUILD | TICK_EMIT) on 100 K subscribers of every AOI kind and 400 K entities over six ticks: statuses and
    error count, every slot's pairs (channel, dist, interval) with a failed or unqueried slot keeping its run, the sub / unsub diff
    as sets and their counts, the carried fan-out state (kept pairs keep last / last_index / flags without PF_NEW, new pairs start
    with PF_NEW | PF_SKIP_SELF, last = now + delay, last_index = 0), and every visible list."""
    e, m = _run_stateful(chd, oracle, use_graphs)
    if use_graphs:
        _FINAL["world"] = (e, m)
    else:
        e.close()


def test_window_exhaustion_refuses_only_queries_that_need_a_window(chd, oracle):
    """The same world with a window scratch of 60 % of what a tick needs: CHD_OVF_WINDOW, required_window_cells = the restated
    total, every query exact or CHD_Q_ERR_CAPACITY, CAPACITY only where the window is not empty (spots-only queries and shapes
    that miss the grid are never refused), the answered windows fit the scratch, refused subscribers keep their pairs and
    fan-out state bit for bit and every other subscriber is updated."""
    from tests._oracle import make_grid

    og = make_grid(*WORLD)
    ticks = _world()[:3]
    cap = int(0.6 * min(int(tk["wn"].sum()) for tk in ticks))
    e = _engine(chd, cap)
    m = Model()
    n_refused = n_spots_only = 0
    for tk in ticks:
        q, slots, t, wn = tk["q"], tk["slots"], tk["t"], tk["wn"]
        e.set_entities(tk["ex"], tk["ez"])
        batch, keep = chd.engine.make_batch(q["n"], sub=slots, **Q.batch_kwargs(q))
        s = chd.capi.TickSummary()
        rc = e.L.chd_tick(e.h, C.byref(batch), t, chd.capi.TICK_BUILD | chd.capi.TICK_EMIT, C.byref(s))
        assert rc == chd.capi.ERR_CAPACITY and s.overflow == chd.capi.OVF_WINDOW, (rc, s.overflow)
        assert s.required_window_cells == int(wn.sum()) > cap
        st, qoff, qch, qdist = oracle.query_batch(og, q["n"], n_threads=_threads(), **Q.batch_kwargs(q))
        gst = e.get_query_status(q["n"])
        refused = gst == chd.capi.Q_ERR_CAPACITY
        bad = np.nonzero(refused & (wn == 0))[0]
        assert len(bad) == 0, ("queries with an empty window refused for capacity", [
            (int(i), "spots only" if q["kind"][i] == Q.AOI_SPOTS else f"kind {int(q['kind'][i])}", int(st[i])) for i in bad[:5]])
        np.testing.assert_array_equal(gst[~refused], st[~refused])
        assert int(wn[~refused].sum()) <= cap
        assert refused.sum() > 1000 and (~refused & (wn > 0)).sum() > 1000
        n_refused += int(refused.sum())
        n_spots_only += int(((wn == 0) & (q["kind"] == Q.AOI_SPOTS) & (st == 0)).sum())
        assert s.n_query_errors == int((gst != 0).sum())
        new, gone, n_kept = m.update(slots, gst == 0, qoff, qch, qdist, t, q["kind"])
        assert (s.n_sub_new, s.n_unsub, s.n_kept) == (len(new), len(gone), n_kept)
        _check_pairs(oracle, e.get_pairs(s.n_pairs), m)
        (ns, nc), (us, uc) = e.get_diff(s.n_sub_new, s.n_unsub)
        np.testing.assert_array_equal(_canon(ns, nc), np.sort(new))
        np.testing.assert_array_equal(_canon(us, uc), np.sort(gone))
        _fanout_between_ticks(e, m, t)
    assert n_refused > 10_000 and n_spots_only > 3_000
    e.close()


def test_adjacent_broadcast_over_scale_state(chd, oracle):
    """chd_adjacent_broadcast over the interest test's final subscriptions (box subscribers spanning 100+ cells, cells with more
    than 32 subscribers): every cell x two filter combinations, random senders and forwarded clients, against
    orc_adjacent_broadcast."""
    from tests._oracle import make_grid, u32p

    if "world" not in _FINAL:
        _FINAL["world"] = _run_stateful(chd, oracle, True)
    e, m = _FINAL.pop("world")
    og = make_grid(*WORLD)
    cells = WORLD[4] * WORLD[5]
    rng = np.random.default_rng(77)
    runs = np.diff(m.off)
    assert (runs[m.box_run] >= 100).sum() > 100  # long runs for the de-duplication scan
    conn = np.arange(1, S + 1, dtype=np.uint32)
    types = rng.integers(1, 3, S).astype(np.uint8)
    e.set_subscriber_types(types)
    sub_of_pair = np.repeat(np.arange(S), runs)
    cell_of_pair = m.f["channel"].astype(np.int64) - S0
    order = np.lexsort((sub_of_pair, cell_of_pair))
    cell_off = np.searchsorted(cell_of_pair[order], np.arange(cells + 1)).astype(np.uint32)
    list_conn = np.ascontiguousarray(conn[sub_of_pair[order]])
    list_type = np.ascontiguousarray(types[sub_of_pair[order]])
    per_cell = np.diff(cell_off.astype(np.int64))
    assert (per_cell > 32).sum() > 1000, per_cell.max()  # one warp's loop over a cell runs more than once
    combos = np.array([64 | 4 | 16, 64 | 8 | 32], np.uint32)
    ch = np.repeat(np.arange(cells, dtype=np.uint32) + S0, 2)
    fl = np.tile(combos, cells)
    M = len(ch)
    snd = np.where(rng.random(M) < 0.8, conn[rng.integers(0, S, M)], 0).astype(np.uint32)
    cli = np.where(rng.random(M) < 0.5, conn[rng.integers(0, S, M)], 0).astype(np.uint32)
    # the oracle, message by message over threads (ctypes releases the GIL)
    ucap = int(per_cell.max()) * 9 + 1

    def run(lo, hi):
        buf = np.zeros(ucap, np.uint32)
        out, cnt = [], np.zeros(hi - lo, np.int64)
        args = (u32p, cell_off, list_conn, list_type)
        for k in range(lo, hi):
            n = oracle.lib.orc_adjacent_broadcast(C.byref(og), int(ch[k]), int(fl[k]), int(snd[k]), int(cli[k]),
                                                  cell_off.ctypes.data_as(args[0]), list_conn.ctypes.data_as(args[0]),
                                                  list_type.ctypes.data, buf.ctypes.data_as(args[0]), ucap)
            cnt[k - lo] = n
            out.append(buf[:n].copy())
        return cnt, np.concatenate(out) if out else np.zeros(0, np.uint32)

    step = 4096
    with cf.ThreadPoolExecutor(_threads()) as ex:
        parts = list(ex.map(lambda lo: run(lo, min(lo + step, M)), range(0, M, step)))
    want_cnt = np.concatenate([p[0] for p in parts])
    want = np.concatenate([p[1] for p in parts])
    want_off = np.concatenate([[0], np.cumsum(want_cnt)])
    got_all = []
    for lo in range(0, M, 16384):
        hi = min(lo + 16384, M)
        st, off, slot = e.adjacent_broadcast(ch[lo:hi], fl[lo:hi], snd[lo:hi], cli[lo:hi], cap=int(want_off[hi] - want_off[lo]) + 1)
        assert (st == 0).all()
        np.testing.assert_array_equal(np.diff(off.astype(np.int64)), want_cnt[lo:hi])
        msg = np.repeat(np.arange(hi - lo), np.diff(off.astype(np.int64)))
        got = conn[slot]
        srt = np.lexsort((got, msg))
        got, msg = got[srt], msg[srt]
        assert not ((np.diff(got.astype(np.int64)) == 0) & (np.diff(msg) == 0)).any(), "a connection was reported twice"
        got_all.append(got)
    np.testing.assert_array_equal(np.concatenate(got_all), want)
    assert len(want) > 10_000_000
    e.close()
