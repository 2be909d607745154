"""Explicit subscriptions on the GPU (chd_apply_subscriptions, include/chd_gpu_subs.h) against the oracle (tests/_subs_oracle.py: the
presence-mask merge of subscription.go:34-125 over the CPU oracle's channels): statuses and pairs after hand-built batches, the fan-out
over explicit pairs with device-owned rings, the interaction with the interest update, a config #2-shaped world (1 M entities,
100 K slots) with random op batches between ticks, the capacity rule, slab engines, and ticks that do not use the feature.
Run on an H100:  python -m pytest tests/test_gpu_subs.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests._subs_oracle import DIST_EXPLICIT, ERR_CAPACITY, OPT_DELAY, OPT_INTERVAL, OPT_SKIP_FIRST, OPT_SKIP_SELF, SubsOracle
from tests.test_gpu_fanout_scale import _due_table
from tests.test_gpu_fetch_delta import DeltaSet
from tests.test_gpu_rings_scale import _assert_rings, _csr, _due_from
from tests.test_oracle_delta import _cells

pytestmark = pytest.mark.gpu

S0 = 65536
MS = 1_000_000
GRID = (-1000.0, -750.0, 100.0, 100.0, 20, 15)  # 300 cells
C_SMALL = 300


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
    ns.torch, ns.capi, ns.engine, ns.L = torch, capi, engine, capi.lib()
    return ns


def _random_ops(rng, n, n_slots, cells, bad=0.0):
    slot = rng.integers(0, n_slots + (2 if bad else 0), n).astype(np.uint32)
    ch = (S0 + rng.integers(0, cells + (3 if bad else 0), n)).astype(np.uint32)
    op = (rng.random(n) < 0.35).astype(np.uint8)
    present = rng.integers(0, 16, n).astype(np.uint8)
    iv = rng.choice(np.array([20, 33, 50, 100, 250], np.uint32), n)
    dl = rng.integers(-5, 60, n).astype(np.int32)
    ss = rng.integers(0, 2, n).astype(np.uint8)
    sf = rng.integers(0, 2, n).astype(np.uint8)
    return slot, ch, op, present, iv, dl, ss, sf


def _apply(e, o, ops, t, max_pairs=None, status=True):
    slot, ch, op, present, iv, dl, ss, sf = ops
    got = e.apply_subscriptions(slot, ch, op, interval=iv, delay=dl, skip_self=ss, skip_first=sf, now_ns=t, present=present, status=status)
    want = o.apply(slot, ch, op, t, present=present, interval=iv, delay=dl, skip_self=ss, skip_first=sf, max_pairs=max_pairs)
    if status:
        np.testing.assert_array_equal(got, want)
    return want


def _check_pairs(e, o, n_slots, state=True):
    """channel, dist, interval, SkipSelf and (state) the fan-out state of every pair against the oracle"""
    p = e.get_pairs()
    w = o.table(n_slots)
    np.testing.assert_array_equal(p["off"], w["off"])
    np.testing.assert_array_equal(p["channel"], w["channel"])
    np.testing.assert_array_equal(p["dist"], w["dist"])
    np.testing.assert_array_equal(p["interval"], w["interval"])
    np.testing.assert_array_equal((p["flags"] & 4).astype(bool), w["skip_self"])
    if state:
        last, had, li = o.state()
        np.testing.assert_array_equal(p["last"], last)
        np.testing.assert_array_equal((p["flags"] & 1).astype(bool), had)
        np.testing.assert_array_equal(p["last_index"], li)
    return p


def _small(chd, n_slots=16, start=None, max_pairs=1 << 14):
    e = chd.engine.Engine(chd.engine.grid_cfg(*GRID), 64, 32, max_pairs=max_pairs, max_due=1 << 16, max_ring_entries=C_SMALL * 1024)
    e.set_entities(np.zeros(1), np.zeros(1))
    conn = np.arange(101, 101 + n_slots, dtype=np.uint32)
    e.set_subscribers(conn)
    if start is not None:
        assert e.L.chd_set_channel_start_times(e.h, chd.capi.ptr(np.ascontiguousarray(start, np.int64))) == chd.capi.OK
    return e, conn


def test_statuses_and_pairs_small_batches(chd, oracle):
    """Repeats on one pair, free slots, a slot with a removal pending, bad channel ids and per-channel start times: every status and
    every pair field equals the oracle's after each batch."""
    rng = np.random.default_rng(1)
    start = rng.integers(0, 5 * MS, C_SMALL).astype(np.int64)
    e, conn = _small(chd, start=start)
    o = SubsOracle(oracle, C_SMALL, conn, default_interval_ms=e.lim.default_fanout_interval_ms,
                   default_delay_ms=e.lim.default_fanout_delay_ms, start_ns=start)
    e.remove_subscribers([3])
    o.pending.add(3)
    A, B = S0 + 7, S0 + 150
    hand = (np.array([0, 0, 0, 0, 0, 1, 1, 3, 20, 2, 2, 4, 4], np.uint32),
            np.array([A, A, A, A, A, A, B, A, A, S0 + 300, 5, B, B], np.uint32),
            np.array([0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0], np.uint8),
            np.array([0, 15, 0, 0, OPT_DELAY | OPT_SKIP_FIRST, OPT_INTERVAL | OPT_SKIP_SELF, 0, 0, 0, 0, 0, 0, OPT_INTERVAL], np.uint8),
            np.full(13, 77, np.uint32), np.full(13, 30, np.int32), np.zeros(13, np.uint8), np.ones(13, np.uint8))
    st = _apply(e, o, hand, 1000 * MS)
    assert list(st) == [0, 1, 2, 3, 0, 0, 0, 4, 4, 5, 5, 3, 0]  # NEW MERGED UNSUB NOT_SUB NEW NEW NEW ERR_SLOT x2 ERR_CHANNEL x2 NOT_SUB NEW
    _check_pairs(e, o, 16)
    for k in range(6):
        _apply(e, o, _random_ops(rng, 40 + 90 * k, 16, C_SMALL, bad=0.1), (1000 + 10 * k) * MS)
        _check_pairs(e, o, 16)
    s = e.summary()
    assert s.n_pairs == len(o.pairs) and s.overflow == 0
    e.close()


def _updates(rng, cells, t_prev, t, conn, flood=0):
    n_cell = rng.integers(0, 4, cells)
    n_cell[:flood] = 100  # (the first `flood` cells: their rings pass 512 entries, and evictions follow maxFanOutIntervalMs)
    n = int(n_cell.sum())
    arr = np.sort(rng.integers(t_prev + 1, t + 1, n)).astype(np.int64)
    cell = np.repeat(np.arange(cells), n_cell)
    arr = arr[np.lexsort((arr, cell))]
    snd = np.where(rng.random(n) < 0.5, rng.choice(conn, n), 7).astype(np.uint32)
    return n_cell, cell.astype(np.uint32), arr, snd


def test_fanout_over_explicit_pairs(chd, oracle):
    """24 ticks of random op batches (delay, SkipFirst, SkipSelf, intervals), device-owned ring updates and chd_fanout_tick: the due
    list equals orc_channels_tick_data's sends as a set, and every pair's state the oracle's.  Four cells get 100 updates a tick, so
    their rings pass 512 entries and drop their oldest entry only when it is older than the cell's maxFanOutIntervalMs (512 entries
    span about 170 ms, so a 250 ms maximum keeps more of them): the rings equal the oracle's every tick only if the device raised that
    maximum exactly when the oracle did (at creation only)."""
    rng = np.random.default_rng(2)
    e, conn = _small(chd)
    e.rings_init(1024)
    o = SubsOracle(oracle, C_SMALL, conn, default_interval_ms=e.lim.default_fanout_interval_ms, default_delay_ms=e.lim.default_fanout_delay_ms)
    t_prev, n_due, longest, maxima = 0, 0, 0, set()
    for tick in range(24):
        t = (tick + 1) * 33 * MS
        _apply(e, o, _random_ops(rng, 200, 16, 40), t)
        n_cell, cell, arr, snd = _updates(rng, C_SMALL, t_prev, t, conn, flood=4)
        e.rings_append(_csr(n_cell), arr, snd)
        o.ch.on_update(cell, arr, snd)
        want_rings = o.ch.get_rings()
        _assert_rings(e.get_rings(), want_rings)
        longest = max(longest, int(np.diff(want_rings["off"].astype(np.int64))[:4].max()))
        maxima |= set(want_rings["max_interval_ms"][:4].tolist())
        e.fanout_tick(t)
        s = e.summary()
        sends, soff = o.ch.tick_data(t, 1 << 16)
        s_cell = np.repeat(np.arange(C_SMALL), np.diff(soff.astype(np.int64)))
        want = _due_table(sends["conn_id"], (s_cell + S0).astype(np.uint32), sends["kind"], sends["n_selected"], sends["first_sel"],
                          sends["last_sel"], sends["sel_hash"], sends["last_message_index"], sends["window_hi"])
        got = _due_from(conn, e.get_due(s.n_due))
        np.testing.assert_array_equal(got, want)
        _check_pairs(e, o, 16)
        n_due += s.n_due
        t_prev = t
    assert n_due > 100
    assert longest > 600 and len(maxima) > 2  # rings the maximum kept above 512, under maxima that grew as subscriptions were created
    e.close()


def test_interest_update_over_explicit_pairs(chd, oracle):
    """A query that misses an explicit cell unsubscribes it (unsub list); one that hits it keeps its flags and fan-out state and takes
    the damping interval and the query's dist; chd_remove_subscribers unsubscribes explicit pairs."""
    e, conn = _small(chd)
    cx, cz = np.array([-1000 + 550.0]), np.array([-750 + 350.0])  # cell (5, 3) = index 65
    A, B = S0 + 200, S0 + 65
    st = e.apply_subscriptions([0, 0, 1], [A, B, A], [0, 0, 0], interval=[400, 400, 400], delay=[25, 25, 25], skip_self=[0, 0, 0],
                               skip_first=[1, 1, 1], now_ns=10 * MS)
    assert list(st) == [0, 0, 0]
    before = e.get_pairs()
    batch, keep = chd.engine.make_batch(1, sub=np.array([0], np.uint32), sphere=(cx, cz, np.array([10.0])))
    qs, qoff, qch, qdist = e.query_channel_ids(batch)
    assert list(qch) == [B]
    e.update_interest(batch, 20 * MS)
    s = e.summary()
    assert (s.n_sub_new, s.n_unsub, s.n_kept) == (0, 1, 1)
    _, (un_sub, un_ch) = e.get_diff(s.n_sub_new, s.n_unsub)
    assert list(un_sub) == [0] and list(un_ch) == [A]
    p = e.get_pairs()
    assert list(p["off"][:3]) == [0, 1, 2] and list(p["channel"]) == [B, A]
    assert p["dist"][0] == qdist[0] and p["interval"][0] == e.L.chd_damping_interval_ms(int(qdist[0]), e.lim.default_fanout_interval_ms)
    k = int(np.nonzero(before["channel"][:2] == B)[0][0])
    assert (p["flags"][0] & 5) == (before["flags"][k] & 5) == 1  # SkipFirst -> hadFirstFanOut, SkipSelf off: kept
    assert p["last"][0] == before["last"][k] == 35 * MS and p["last_index"][0] == 0
    assert p["dist"][1] == DIST_EXPLICIT and p["interval"][1] == 400
    e.remove_subscribers([1])
    e.update_interest(chd.engine.make_batch(0)[0], 30 * MS)
    s = e.summary()
    _, (un_sub, un_ch) = e.get_diff(s.n_sub_new, s.n_unsub)
    assert list(un_sub) == [1] and list(un_ch) == [A] and s.n_pairs == 1
    # the removed slot is free: ops on it are refused
    assert list(e.apply_subscriptions([1], [A], [0], now_ns=40 * MS)) == [chd.capi.SUB_ERR_SLOT]
    e.close()


def test_capacity_is_transactional(chd, oracle):
    """A batch that would exceed max_pairs applies nothing: every valid op gets ERR_CAPACITY, the next summary carries CHD_OVF_PAIRS and
    required_pairs, and the batches and ticks (interest update + fan-out) after it match the oracle."""
    rng = np.random.default_rng(3)
    e, conn = _small(chd, max_pairs=64)
    o = SubsOracle(oracle, C_SMALL, conn, default_interval_ms=e.lim.default_fanout_interval_ms, default_delay_ms=e.lim.default_fanout_delay_ms)
    ops = (np.repeat(np.arange(16, dtype=np.uint32), 3), (S0 + np.tile(np.arange(3), 16)).astype(np.uint32), np.zeros(48, np.uint8),
           np.zeros(48, np.uint8), None, None, None, None)
    _apply(e, o, ops, MS, max_pairs=64)
    big = (np.arange(20, dtype=np.uint32) % 16, (S0 + 100 + np.arange(20)).astype(np.uint32), np.zeros(20, np.uint8), np.zeros(20, np.uint8),
           None, None, None, None)
    big = (np.append(big[0], 99).astype(np.uint32), np.append(big[1], S0).astype(np.uint32), np.append(big[2], 0).astype(np.uint8),
           np.append(big[3], 0).astype(np.uint8), None, None, None, None)
    st = _apply(e, o, big, 2 * MS, max_pairs=64)
    assert (st[:20] == ERR_CAPACITY).all() and st[20] == chd.capi.SUB_ERR_SLOT
    with pytest.raises(chd.capi.ChdError):
        e.summary()
    h = e.h
    from channeld_b200.capi import TickSummary
    import ctypes as C

    s = TickSummary()
    # the overflow bit was read (and cleared) by the summary above; the counters it left say what was needed
    assert e.L.chd_summary(h, C.byref(s)) == chd.capi.OK and s.n_pairs == 48 and s.required_pairs == 68
    _check_pairs(e, o, 16)
    from tests import _oracle

    g = _oracle.make_grid(*GRID)
    damp = lambda d: oracle.damping(d, e.lim.default_fanout_interval_ms)  # noqa: E731
    for k in range(4):
        t = (3 + k) * MS
        _apply(e, o, _random_ops(rng, 30, 16, 8), t, max_pairs=64)
        _check_pairs(e, o, 16)
        # one sphere inside one cell each, for the two slots with the most pairs: a run shrinks to one pair, the total never grows
        qs = np.array(sorted(sorted(range(16), key=lambda sl: -len(o.cells_of.get(sl, ())))[:2]), np.uint32)
        cx, cz, r = -1000 + 50.0 + 100.0 * qs, np.full(2, -700.0), np.full(2, 10.0)
        batch, keep = chd.engine.make_batch(2, sub=qs, sphere=(cx, cz, r))
        q_st, q_off, q_ids, q_dist = oracle.query_batch(g, 2, sphere=(cx, cz, r))
        s = e.tick(batch, t + MS // 2, chd.capi.TICK_ALL)
        for j, sl in enumerate(qs.tolist()):
            o.interest(sl, q_ids[q_off[j]:q_off[j + 1]].astype(np.int64) - S0, q_dist[q_off[j]:q_off[j + 1]], t + MS // 2, damp)
        assert s.overflow == 0 and s.n_pairs == len(o.pairs) <= 64
        _check_pairs(e, o, 16)
    e.close()


def test_slab_engine_refuses(chd):
    e, conn = _small(chd)
    e.set_slab(0, 10, 1)
    st = e.L.chd_apply_subscriptions(e.h, chd.capi.SubBatch(n=0), 0, None)
    assert st == chd.capi.ERR_STATE
    with pytest.raises(chd.capi.ChdError) as ex:
        e.apply_subscriptions([0], [S0], [0])
    assert ex.value.status == chd.capi.ERR_STATE
    e.close()


def test_refused_while_interest_is_pending(chd):
    e, conn = _small(chd)
    batch, keep = chd.engine.make_batch(1, sub=np.array([0], np.uint32), sphere=(np.array([0.0]), np.array([0.0]), np.array([10.0])))
    e.begin_interest(batch, MS, with_fanout=False)
    with pytest.raises(chd.capi.ChdError) as ex:
        e.apply_subscriptions([0], [S0], [0])
    assert ex.value.status == chd.capi.ERR_STATE
    e.tick(None, MS, chd.capi.TICK_BUILD)
    assert list(e.apply_subscriptions([0], [S0], [0], now_ns=MS)) == [0]
    e.close()


def test_ticks_without_the_feature_launch_the_same(chd):
    """A tick sequence launches the same kernels and graphs whether or not explicit ops were applied before it started."""
    counts = []
    for with_ops in (False, True):
        e, conn = _small(chd)
        rng = np.random.default_rng(4)
        cx, cz = -1000 + rng.random(16) * 2000, -750 + rng.random(16) * 1500
        batch, keep = chd.engine.make_batch(16, sub=np.arange(16, dtype=np.uint32), sphere=(cx, cz, np.full(16, 120.0)))
        for k in range(6):  # warm-up: both pair-buffer parities captured
            e.tick(batch, (k + 1) * 33 * MS, chd.capi.TICK_ALL)
        if with_ops:
            e.apply_subscriptions([0, 1, 2], [S0 + 1, S0 + 2, S0 + 3], [0, 0, 0], now_ns=7 * 33 * MS)
            e.apply_subscriptions([0], [S0 + 9], [0], now_ns=7 * 33 * MS)
        l0, g0 = e.launch_count(), e.graph_launch_count()
        for k in range(6, 14):
            e.tick(batch, (k + 1) * 33 * MS, chd.capi.TICK_ALL)
        counts.append((e.launch_count() - l0, e.graph_launch_count() - g0))
        e.close()
    assert counts[0] == counts[1], counts


# ---- config #2 shape: 1 M entities, 100 K slots, 225 cells

def _scale_world(chd):
    from channeld_b200 import synth

    wc = synth.CONFIGS["benchmark"]
    ex, ez = synth.entities(wc)
    conn, cx, cz, r = synth.subscribers(wc, ex, ez, 50.0)
    return wc, ex, ez, conn.astype(np.uint32), cx, cz, r


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_scale_ops_queries_and_fanout(chd, oracle, graphs):
    """30 ticks at config #2's shape: each tick a random op batch (up to 200 K ops) applied between ticks, a query batch for a random
    tenth of the slots and chd_tick(TICK_ALL) with device-owned rings.  Every tick: the pair state, the due list and the expanded visible
    lists of a 1 % slot sample equal the oracle's."""
    from tests import _oracle

    wc, ex, ez, conn, cx, cz, r = _scale_world(chd)
    S, C = len(conn), wc.cols * wc.rows
    e = chd.engine.Engine(wc.cfg(), len(ex), S, max_pairs=3 << 20, max_due=1 << 22, max_ring_entries=C * 1024,
                          max_visible=3_000_000_000)
    e.enable_graphs(graphs)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    e.rings_init(1024)
    g = _oracle.make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)
    o = SubsOracle(oracle, C, conn, default_interval_ms=e.lim.default_fanout_interval_ms, default_delay_ms=e.lim.default_fanout_delay_ms)
    damp = lambda d: oracle.damping(d, e.lim.default_fanout_interval_ms)  # noqa: E731
    rng = np.random.default_rng(6)
    sizes = [200_000 if k == 17 else int(rng.integers(1, 20_000)) for k in range(30)]
    t_prev = 0
    for tick in range(30):
        t = (tick + 1) * 33 * MS
        if tick:
            _apply(e, o, _random_ops(rng, sizes[tick], S, C), t - MS)
        qs = np.arange(S, dtype=np.uint32) if tick == 0 else np.sort(rng.choice(S, S // 10, replace=False)).astype(np.uint32)
        qr = r[qs] * rng.choice([0.5, 1.0, 2.0, 3.0], len(qs))
        batch, keep = chd.engine.make_batch(len(qs), sub=qs, sphere=(cx[qs], cz[qs], qr))
        q_st, q_off, q_ids, q_dist = oracle.query_batch(g, len(qs), sphere=(cx[qs], cz[qs], qr))
        n_cell, cell, arr, snd = _updates(rng, C, t_prev, t, conn[:64])
        e.rings_append(_csr(n_cell), arr, snd)
        s = e.tick(batch, t, chd.capi.TICK_ALL)
        # the oracle in the engine's order: interest update, ring updates, tickData
        qoff = q_off.astype(np.int64)
        for k, sl in enumerate(qs.tolist()):
            if q_st[k] == 0:
                o.interest(sl, q_ids[qoff[k]:qoff[k + 1]].astype(np.int64) - S0, q_dist[qoff[k]:qoff[k + 1]], t, damp)
        o.ch.on_update(cell, arr, snd)
        sends, soff = o.ch.tick_data(t, 1 << 22)
        s_cell = np.repeat(np.arange(C), np.diff(soff.astype(np.int64)))
        want = _due_table(sends["conn_id"], (s_cell + S0).astype(np.uint32), sends["kind"], sends["n_selected"], sends["first_sel"],
                          sends["last_sel"], sends["sel_hash"], sends["last_message_index"], sends["window_hi"])
        assert s.overflow == 0 and s.n_pairs == len(o.pairs)
        np.testing.assert_array_equal(_due_from(conn, e.get_due(s.n_due)), want)
        p = _check_pairs(e, o, S, state=tick % 5 == 4)
        cs, se = e.get_cells()
        for sl in rng.choice(S, S // 100, replace=False).tolist():
            cells = p["channel"][p["off"][sl]:p["off"][sl + 1]].astype(np.int64) - S0
            vis = np.concatenate([se[cs[c]:cs[c + 1]] for c in cells]) if len(cells) else np.zeros(0, np.uint32)
            np.testing.assert_array_equal(e.get_visible_slot(sl), vis)
        t_prev = t
    e.close()


class _FetchSet:
    """One set of pinned read-back buffers for chd_fetch_results_async_delta: the pairs (offsets, channel, dist, interval), the due
    list and the visible delta, sentinel-filled before each use."""

    def __init__(self, chd, S, P, D, delta_cap):
        t = chd.torch
        self.off = t.zeros(S + 1, dtype=t.int32).pin_memory()
        self.ch, self.dist, self.iv = (t.zeros(P, dtype=t.int32).pin_memory() for _ in range(3))
        self.due = t.zeros(D * 12, dtype=t.int32).pin_memory()  # 48 B per decision
        self.r = chd.capi.ResultBuffers()
        p = chd.capi.ptr
        self.r.pair_off, self.r.pair_channel, self.r.pair_dist, self.r.pair_interval_ms = p(self.off), p(self.ch), p(self.dist), p(self.iv)
        self.r.pair_cap, self.r.due, self.r.due_cap = P, p(self.due), D
        self.ds = DeltaSet(chd, S + 1, delta_cap)

    def reset(self):
        for a in (self.off, self.ch, self.dist, self.iv, self.due):
            a.fill_(-1)
        self.ds.reset()

    def fetch(self, chd, e):
        return chd.L.chd_fetch_results_async_delta(e.h, C.byref(self.r), C.byref(self.ds.b), chd.capi.ptr(self.ds.hdr))

    def check(self, chd, conn, s, c, want, k):
        P, nd = int(s.n_pairs), int(s.n_due)
        assert s.overflow == 0 and P == len(want["channel"]), k
        np.testing.assert_array_equal(self.off.numpy().view(np.uint32), want["off"], err_msg="tick %d pair_off" % k)
        for name, buf in (("channel", self.ch), ("dist", self.dist), ("interval", self.iv)):
            np.testing.assert_array_equal(buf.numpy()[:P].view(np.uint32), want[name], err_msg="tick %d %s" % (k, name))
        due = self.due.numpy()[:nd * 12].view(chd.capi.DUE_DTYPE)
        np.testing.assert_array_equal(_due_from(conn, due), want["due"], err_msg="tick %d due" % k)
        for name, u, v in zip(("enter_off", "enter", "leave_off", "leave"), self.ds.lists(c), want["delta"]):
            np.testing.assert_array_equal(u, v, err_msg="tick %d delta %s" % (k, name))


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
def test_scale_pipelined_with_visible_delta(chd, oracle, graphs):
    """The pipelined two-stream loop at config #2's slot and pair counts (100 K slots, 225 cells; 100 K entities, so that the index-mode
    visible delta of every tick, the first one included, stays small enough to check in full): per tick a random op batch (up to
    200 K ops, no host synchronisation) applied while the previous tick is still in flight, a query batch for a tenth of the slots,
    chd_tick(TICK_ALL | TICK_VISIBLE_DELTA) and chd_fetch_results_async_delta into one of two pinned buffer sets; then chd_fetch_wait for
    the previous tick.  Its pairs, due list and visible delta must equal the oracle's state of that tick, although ops and a tick have
    been enqueued since: what was fetched stays intact."""
    from channeld_b200 import synth
    from tests import _oracle

    wc = synth.scaled(synth.CONFIGS["benchmark"], 100_000, 100_000)
    ex, ez = synth.entities(wc)
    conn, cx, cz, r = synth.subscribers(wc, ex, ez, 50.0)
    conn = conn.astype(np.uint32)
    S, NC, P, D = len(conn), wc.cols * wc.rows, 3 << 20, 1 << 21
    e = chd.engine.Engine(wc.cfg(), len(ex), S, max_pairs=P, max_due=D, max_ring_entries=NC * 1024, max_visible=1 << 29)
    e.enable_graphs(graphs)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    e.reserve_visible_delta(1 << 26)
    e.rings_init(1024)
    g = _oracle.make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)
    ent_cell = _cells(oracle, g, ex, ez)
    o = SubsOracle(oracle, NC, conn, default_interval_ms=e.lim.default_fanout_interval_ms, default_delay_ms=e.lim.default_fanout_delay_ms)
    damp = lambda d: oracle.damping(d, e.lim.default_fanout_interval_ms)  # noqa: E731
    rng = np.random.default_rng(7)
    sizes = [200_000 if k == 11 else int(rng.integers(1, 20_000)) for k in range(30)]
    sets = [_FetchSet(chd, S, P, D, 1 << 26) for _ in range(2)]
    prev_state = (np.zeros(0, np.uint32), np.zeros(1, np.uint64), np.zeros(0, np.uint32))
    pending = []
    t_prev = 0
    for tick in range(31):
        if tick < 30:
            t = (tick + 1) * 33 * MS
            if tick:  # between ticks: the previous tick and its read-back are still in flight
                slot, ch, op, present, iv, dl, ss, sf = _random_ops(rng, sizes[tick], S, NC)
                assert e.apply_subscriptions(slot, ch, op, interval=iv, delay=dl, skip_self=ss, skip_first=sf, now_ns=t - MS, present=present,
                                             status=False) is None
                o.apply(slot, ch, op, t - MS, present=present, interval=iv, delay=dl, skip_self=ss, skip_first=sf)
            qs = np.arange(S, dtype=np.uint32) if tick == 0 else np.sort(rng.choice(S, S // 10, replace=False)).astype(np.uint32)
            qr = r[qs] * rng.choice([0.5, 1.0, 2.0, 3.0], len(qs))
            batch, keep = chd.engine.make_batch(len(qs), sub=qs, sphere=(cx[qs], cz[qs], qr))
            n_cell, cell, arr, snd = _updates(rng, NC, t_prev, t, conn[:64])
            e.rings_append(_csr(n_cell), arr, snd)
            fs = sets[tick % 2]
            fs.reset()
            assert chd.L.chd_tick(e.h, C.byref(batch), t, chd.capi.TICK_ALL | chd.capi.TICK_VISIBLE_DELTA, None) == 0, chd.L.chd_last_error(e.h)
            assert fs.fetch(chd, e) == 0, chd.L.chd_last_error(e.h)
            # the oracle's state of this tick: interest update, ring updates, tickData, the delta against the previous tick's pairs
            q_st, q_off, q_ids, q_dist = oracle.query_batch(g, len(qs), sphere=(cx[qs], cz[qs], qr))
            qoff = q_off.astype(np.int64)
            for k, sl in enumerate(qs.tolist()):
                if q_st[k] == 0:
                    o.interest(sl, q_ids[qoff[k]:qoff[k + 1]].astype(np.int64) - S0, q_dist[qoff[k]:qoff[k + 1]], t, damp)
            o.ch.on_update(cell, arr, snd)
            sends, soff = o.ch.tick_data(t, 1 << 22)
            s_cell = np.repeat(np.arange(NC), np.diff(soff.astype(np.int64)))
            want = o.table(S)
            want["due"] = _due_table(sends["conn_id"], (s_cell + S0).astype(np.uint32), sends["kind"], sends["n_selected"], sends["first_sel"],
                                     sends["last_sel"], sends["sel_hash"], sends["last_message_index"], sends["window_hi"])
            now_state = (ent_cell, want["off"].astype(np.uint64), (want["channel"].astype(np.int64) - S0).astype(np.uint32))
            want["delta"] = oracle.visible_delta(NC, prev_state, now_state)
            prev_state = now_state
            pending.append((tick, fs, want))
            t_prev = t
        if tick == 0:
            continue
        k, fs, want = pending.pop(0)
        s, c = chd.capi.TickSummary(), chd.capi.DeltaCounts()
        assert chd.L.chd_fetch_wait_delta(e.h, C.byref(s), C.byref(c)) == 0, chd.L.chd_last_error(e.h)
        fs.check(chd, conn, s, c, want, k)
    e.close()
