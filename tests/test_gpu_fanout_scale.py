"""The interest diff, the pair grouping by cell and the fan-out pass at the sizes where their kernels change path, against the
oracle's literal emulation of Channel.tickData (one oracle channel per cell, fed the same subscriptions and update rings).

Paths each case is built to take (and asserts it takes):
  grid     cells   pair grouping                  entity build
  a        225     1 pass, 256 bins               1 pass, 256 bins     (the benchmark grid, > 16 x SMs x 128 live pairs)
  b        300     1 pass, 1024 bins              1 pass, 1024 bins
  c        1024    1 pass, 1024 bins              2 passes
  d        1025    2 passes of 256 bins           2 passes
  e        65536   2 passes of 256 bins           2 passes
  f        65792   2 passes, first with 1024 bins 2 passes
every grid at pair capacity 2^21 (plain scatter) and 2^21 + 1 (shared-memory reordered scatter); fan-out blocks whose ring span
is exactly FANOUT_STAGE (640, staged in shared memory) and FANOUT_STAGE + 1 (read from global memory) in the "stage" case.
Run on an H100:  python -m pytest tests/test_gpu_fanout_scale.py -m gpu
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S0 = 65536
MS = 1_000_000
FANOUT_STAGE = 640  # chd_fanout.cuh
FANOUT_BLOCK = 128
SCATTER_REORDER_ABOVE = 2 << 20  # chd_entities.cu: sort passes over more keys than this reorder each tile in shared memory
N_TICKS = 6

GRIDS = {  # offx, offz, w, h, cols, rows
    "a": (-15000.0, -15000.0, 2000.0, 2000.0, 15, 15),
    "b": (-1000.0, -750.0, 100.0, 100.0, 20, 15),
    "c": (-1600.0, -1600.0, 100.0, 100.0, 32, 32),
    "d": (-2050.0, -1250.0, 100.0, 100.0, 41, 25),
    "e": (-12800.0, -12800.0, 100.0, 100.0, 256, 256),
    "f": (-12850.0, -12800.0, 100.0, 100.0, 257, 256),
}
RADII = {"a": (50.0, 1500.0, 2500.0)}  # the benchmark grid with larger radii: more than 3 pairs per subscriber
CAPS = (SCATTER_REORDER_ABOVE, SCATTER_REORDER_ABOVE + 1)

CASES = [pytest.param(g, cap, True, False, id="%s-cap%s" % (g, "plain" if cap == CAPS[0] else "reorder")) for g in GRIDS for cap in CAPS]
CASES += [pytest.param("a", CAPS[0], False, False, id="a-nographs"), pytest.param("b", CAPS[1], True, True, id="b-stage")]


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
    ns.sms = torch.cuda.get_device_properties(0).multi_processor_count
    return ns


def _pair_keys(sub, cell):
    return (np.asarray(sub, np.int64) << 20) | np.asarray(cell, np.int64)


def _intervals(dist):
    return np.select([dist == 0, dist == 1, dist == 2], [20, 50, 100], 20).astype(np.uint32)  # message_spatial.go:16-38


def _due_table(conn, channel, kind, n, first, last, h, li, hi):
    t = np.zeros(len(conn), [("conn", "<u4"), ("channel", "<u4"), ("kind", "<u4"), ("n", "<u4"), ("first", "<u4"), ("last", "<u4"),
                             ("hash", "<u8"), ("last_index", "<u8"), ("window_hi", "<i8")])
    for k, v in zip(t.dtype.names, (conn, channel, kind, n, first, last, h, li, hi)):
        t[k] = v
    return np.sort(t)


def _block_spans(cell_sorted, ring_off):
    """Ring span of every fan-out block: by_cell is the pairs sorted stably by cell, 128 per block iteration; a block stages
    ring_off[first cell] .. ring_off[last cell + 1]."""
    lo = cell_sorted[::FANOUT_BLOCK]
    hi = cell_sorted[FANOUT_BLOCK - 1::FANOUT_BLOCK]
    if len(hi) < len(lo):
        hi = np.concatenate([hi, cell_sorted[-1:]])
    return ring_off[hi + 1].astype(np.int64) - ring_off[lo].astype(np.int64), hi - lo


@pytest.mark.parametrize("grid,cap,graphs,stage", CASES)
def test_fanout_scale_parity(chd, oracle, grid, cap, graphs, stage):
    from tests._oracle import make_grid

    g = GRIDS[grid]
    offx, offz, w, h, cols, rows = g
    C = cols * rows
    W, H = w * cols, h * rows
    og = make_grid(*g)
    rng = np.random.default_rng(1000 + C + cap % 7 + 3 * stage)
    S = 100_000
    conn = np.arange(1, S + 1, dtype=np.uint32)
    ux = rng.random(S)
    if stage:  # sparse columns on the right, so that some blocks cover more than two cells
        ux = np.where(rng.random(S) < 0.98, ux * 0.6, ux)
    cx, cz = offx + ux * W, offz + rng.random(S) * H
    rad = rng.choice(RADII.get(grid, (50.0, 60.0, 120.0)), S)
    ex, ez = np.array([offx + 1.0]), np.array([offz + 1.0])  # fan-out does not depend on entities

    e = chd.engine.Engine(chd.engine.grid_cfg(*g), 1, S, max_pairs=cap, max_due=4 * cap, max_ring_entries=C * 64 + (1 << 17),
                          max_window_cells=S * 32 + 65536)
    e.enable_graphs(graphs)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    e.build()
    chans = oracle.channels(C)
    # the engine's ring CSR, kept in insertion order per cell (= the oracle channels' updateMsgBuffer; never over 512 entries)
    r_cell = np.zeros(0, np.uint32); r_arr = np.zeros(0, np.int64); r_snd = np.zeros(0, np.uint32); r_idx = np.zeros(0, np.uint64)
    msg_index = np.zeros(C, np.uint64)
    bench_state = None
    prev_keys = np.zeros(0, np.int64)
    t = 0
    total_due = total_multi = total_update = 0
    max_live = 0
    spans_seen, multi_cell_block, one_cell_block = set(), False, False
    for tick in range(N_TICKS):
        gap = 70 * MS if tick % 3 == 0 else 33 * MS  # irregular ticks: 20 ms pairs fall up to three intervals behind
        t += gap
        if tick:
            mv = rng.random(S) < 0.3
            cx[mv] = np.clip(cx[mv] + rng.uniform(-0.6, 0.6, mv.sum()) * w, offx + 1e-3, offx + W - 1e-3)
            cz[mv] = np.clip(cz[mv] + rng.uniform(-0.6, 0.6, mv.sum()) * h, offz + 1e-3, offz + H - 1e-3)
        # ---- interest: every subscriber sends its query (identity batch)
        want = oracle.sphere_tick(og, ex, ez, cx, cz, rad)
        assert (want["status"] == 0).all()
        P = len(want["pair_cell"])
        assert P <= cap
        w_sub = np.repeat(np.arange(S), np.diff(want["pair_off"].astype(np.int64)))
        w_cell = want["pair_cell"].astype(np.int64) - S0
        w_iv = _intervals(want["pair_dist"])
        keys = _pair_keys(w_sub, w_cell)
        batch, keep = chd.engine.make_batch(S, sub=None, sphere=(cx, cz, rad))
        e.update_interest(batch, t)
        s = e.summary()
        want_new = np.setdiff1d(keys, prev_keys)
        want_gone = np.setdiff1d(prev_keys, keys)
        n_kept = len(keys) - len(want_new)
        assert (s.n_pairs, s.n_query_errors, s.n_sub_new, s.n_unsub, s.n_kept, s.overflow) == (P, 0, len(want_new), len(want_gone), n_kept, 0)
        (new_s, new_c), (un_s, un_c) = e.get_diff(s.n_sub_new, s.n_unsub)
        np.testing.assert_array_equal(np.sort(_pair_keys(new_s, new_c.astype(np.int64) - S0)), want_new)
        np.testing.assert_array_equal(np.sort(_pair_keys(un_s, un_c.astype(np.int64) - S0)), want_gone)
        pairs = e.get_pairs()
        np.testing.assert_array_equal(pairs["off"].astype(np.uint64), want["pair_off"])
        g_sub = np.repeat(np.arange(S), np.diff(pairs["off"].astype(np.int64)))
        go = np.lexsort((pairs["channel"], g_sub))
        wo = np.lexsort((w_cell, w_sub))
        np.testing.assert_array_equal(pairs["channel"][go].astype(np.int64) - S0, w_cell[wo])
        np.testing.assert_array_equal(pairs["dist"][go], want["pair_dist"][wo])
        np.testing.assert_array_equal(pairs["interval"][go], w_iv[wo])
        # the oracle channels: unsubscribe what left, (re)subscribe what is wanted (existing ones: options merged)
        chans.unsubscribe(want_gone & 0xFFFFF, conn[want_gone >> 20])
        chans.subscribe(w_cell, conn[w_sub], t, w_iv)
        prev_keys = np.sort(keys)
        max_live = max(max_live, P)
        # ---- update rings
        if stage:
            if tick == 0:  # rings fixed for the whole run: 320, 320, 321 entries per cell, arrivals over the whole run
                lens = np.where(np.arange(C) % 3 == 2, 321, 320)
                n_cell = lens
            else:
                n_cell = np.zeros(C, np.int64)
        elif grid == "a":  # bench.py's generator (synth.update_rings): 8 updates per cell per tick, senders are connection ids
            bench_state, _, _, _, _, _ = chd.synth.update_rings(chd.synth.CONFIGS["benchmark"], tick, t, gap, 8, S, ring_len=512,
                                                               state=bench_state)
            n_cell = np.full(C, 8)
        else:
            n_cell = rng.integers(0, 9, C)
        n_new = int(n_cell.sum())
        u_cell = np.repeat(np.arange(C, dtype=np.uint32), n_cell)
        if grid == "a" and not stage:
            u_arr = bench_state["arrival"][:, -8:].reshape(-1)
            u_snd = bench_state["sender"][:, -8:].reshape(-1)
        else:
            span = (N_TICKS * 40 * MS) if stage else 80 * MS
            u_arr = t - rng.integers(0, span // MS, n_new) * MS + (N_TICKS * 40 * MS if stage else 0)  # not time-sorted
            # half the updates come from a connection subscribed to the cell (SkipSelfUpdateFanOut), half from elsewhere
            bc = np.sort(w_cell, kind="stable")
            bs = w_sub[np.argsort(w_cell, kind="stable")]
            cs = np.searchsorted(bc, np.arange(C + 1))
            cnt = np.diff(cs)[u_cell]
            pick = cs[u_cell] + (rng.random(n_new) * np.maximum(cnt, 1)).astype(np.int64)
            u_snd = np.where((rng.random(n_new) < 0.5) & (cnt > 0), conn[bs[np.minimum(pick, len(bs) - 1)]], 7).astype(np.uint32)
        order = np.argsort(u_cell, kind="stable")
        u_cell, u_arr, u_snd = u_cell[order], np.asarray(u_arr, np.int64)[order], np.asarray(u_snd, np.uint32)[order]
        first_idx = np.concatenate([[0], np.cumsum(n_cell)[:-1]])
        u_idx = msg_index[u_cell] + 1 + (np.arange(n_new) - first_idx[u_cell]).astype(np.uint64)
        msg_index += n_cell.astype(np.uint64)
        chans.on_update(u_cell, u_arr, u_snd)
        r_cell = np.concatenate([r_cell, u_cell]); r_arr = np.concatenate([r_arr, u_arr])
        r_snd = np.concatenate([r_snd, u_snd]); r_idx = np.concatenate([r_idx, u_idx])
        o = np.argsort(r_cell, kind="stable")
        r_cell, r_arr, r_snd, r_idx = r_cell[o], r_arr[o], r_snd[o], r_idx[o]
        ring_off = np.searchsorted(r_cell, np.arange(C + 1)).astype(np.uint32)
        assert np.diff(ring_off).max() <= 512  # the oracle's eviction (data.go:166-172) never fires
        if grid == "a" and not stage:
            np.testing.assert_array_equal(r_arr, bench_state["arrival"].reshape(-1))
            np.testing.assert_array_equal(r_idx, bench_state["index"].reshape(-1))
        e.set_rings(ring_off, r_arr, r_snd, r_idx, msg_index)
        spans, ncell = _block_spans(np.sort(w_cell), ring_off)
        spans_seen |= set(spans.tolist())
        multi_cell_block |= bool((ncell >= 2).any())
        one_cell_block |= bool((ncell == 0).any())
        # ---- fan-out
        e.fanout_tick(t)
        s = e.summary()
        assert s.overflow == 0
        sends, soff = chans.tick_data(t, 4 * P + 4096)
        assert s.n_due == len(sends)
        due = e.get_due(s.n_due)
        s_chan = np.repeat(np.arange(C, dtype=np.uint32), np.diff(soff.astype(np.int64))) + S0
        want_due = _due_table(sends["conn_id"], s_chan, sends["kind"], sends["n_selected"], sends["first_sel"], sends["last_sel"],
                              sends["sel_hash"], sends["last_message_index"], sends["window_hi"])
        got_due = _due_table(conn[due["sub"]], due["channel_id"], due["kind"], due["n_selected"], due["first_sel"], due["last_sel"],
                             due["sel_hash"], due["last_message_index"], due["window_hi"])
        np.testing.assert_array_equal(got_due, want_due)
        # committed state of every pair against the oracle's fanOutConnection
        pairs = e.get_pairs()
        g_sub = np.repeat(np.arange(S), np.diff(pairs["off"].astype(np.int64)))
        last, had, li, found = chans.state(pairs["channel"].astype(np.int64) - S0, conn[g_sub])
        assert found.all()
        np.testing.assert_array_equal(pairs["last"], last)
        np.testing.assert_array_equal((pairs["flags"] & 1).astype(bool), had)
        np.testing.assert_array_equal(pairs["last_index"], li)
        total_due += len(sends)
        k = sends["conn_id"].astype(np.int64) * (C + 1) + np.repeat(np.arange(C), np.diff(soff.astype(np.int64)))
        total_multi += int((np.unique(k, return_counts=True)[1] > 2).sum())  # pairs with more than FANOUT_SLOTS decisions
        total_update += int((sends["kind"] == 1).sum())
    # every case runs the paths it is named for
    assert total_due > 100_000 and total_multi > 1000 and total_update > 1000
    if grid == "a":
        assert max_live > 16 * chd.sms * FANOUT_BLOCK, (max_live, chd.sms)  # the fan-out's grid-stride loop runs a second iteration
    if stage:
        assert FANOUT_STAGE in spans_seen and FANOUT_STAGE + 1 in spans_seen and multi_cell_block and one_cell_block
        assert max(spans_seen) > FANOUT_STAGE + 1 and min(spans_seen) < FANOUT_STAGE
