"""Visible-set deltas read back with the tick's other results: chd_fetch_results_async_delta + chd_fetch_wait_delta in the pipelined
loop (tick k's lists copied while tick k+1 runs) and chd_fetch_results_delta, checked against the oracle's set-difference delta
(orc_visible_delta) with the bookkeeping of test_gpu_delta_scale.py.

Every comparison is exact.  In id mode the lists are compared per slot as sets (sorted slot << 32 | id keys): inside a cell the id-mode
lists follow the cell CSR, whose order the oracle does not model.

Constants the copy-loop sizes depend on (SM count from torch):
  COPY_THREADS = 256     chd_results.cu: block size of bulk_copy_kernel
  bulk_copy_grid         chd_results.cu: per segment at most 2 x SMs blocks in hop 1 (HBM staging) and SMs / 4 in hop 2 (pinned
                         host), one 16-byte vector (4 words) per thread and pass; sizes past hop 1's pass loop in both hops
Run on an H100:  python -m pytest tests/test_gpu_fetch_delta.py -m gpu
"""
import ctypes as C
from contextlib import closing

import numpy as np
import pytest

from tests._oracle import make_grid
from tests.test_gpu_sharded_delta import _keys
from tests.test_oracle_delta import _cells

pytestmark = pytest.mark.gpu

MS = 1_000_000
S0 = 0x10000
ID_SPACE = 1 << 21
COPY_THREADS = 256
SENT32, SENT64 = 0x7EADBEEF, 0x7EADBEEF7EADBEEF


@pytest.fixture(scope="module")
def chd():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from channeld_b200 import capi, engine, synth

    class NS:
        pass

    ns = NS()
    ns.torch, ns.capi, ns.engine, ns.synth, ns.L = torch, capi, engine, synth, capi.lib()
    ns.sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns.copy_pass_words = 2 * ns.sms * COPY_THREADS * 4  # words one pass of the largest copy grid moves per segment
    return ns


class DeltaSet:
    """One set of pinned delta buffers (sentinel-filled), its chd_delta_buffers and a pinned fetch header."""

    def __init__(self, chd, slot_cap, entity_cap, shift=0):
        t = chd.torch
        self.eo, self.lo = (t.full((slot_cap + shift,), SENT64, dtype=t.int64).pin_memory() for _ in range(2))
        self.en, self.le = (t.full((entity_cap + shift,), SENT32, dtype=t.int32).pin_memory() for _ in range(2))
        self.hdr = t.zeros(64, dtype=t.int32).pin_memory()
        self.b = chd.capi.DeltaBuffers()
        # shift > 0: every destination one element past its allocation's alignment (the copy's unaligned path)
        p = chd.capi.ptr
        self.b.enter_off, self.b.leave_off = p(self.eo) + 8 * shift, p(self.lo) + 8 * shift
        self.b.enter_entity, self.b.leave_entity = p(self.en) + 4 * shift, p(self.le) + 4 * shift
        self.b.slot_cap, self.b.entity_cap = slot_cap, entity_cap
        self.shift = shift

    def reset(self):
        for a, v in ((self.eo, SENT64), (self.lo, SENT64), (self.en, SENT32), (self.le, SENT32)):
            a.fill_(v)

    def lists(self, c):
        s = self.shift
        k = c.n_slots + 1
        eo, lo = self.eo.numpy()[s:s + k].view(np.uint64), self.lo.numpy()[s:s + k].view(np.uint64)
        return eo.copy(), self.en.numpy()[s:s + c.n_entered].view(np.uint32).copy(), lo.copy(), self.le.numpy()[s:s + c.n_left].view(np.uint32).copy()

    def untouched(self):
        return bool((self.eo.numpy() == SENT64).all() and (self.lo.numpy() == SENT64).all() and (self.en.numpy() == SENT32).all()
                    and (self.le.numpy() == SENT32).all())


class World:
    """A scaled benchmark world whose subscribers stand on entities; `mode` index / id (a random injection into [0, 2^21) as global
    ids) / table (ids spawned in entity order, so table slot i is entity i).  step(k) -> this tick's oracle state."""

    def __init__(self, chd, oracle, mode, N, S, graphs=True, cap=1 << 24, step=150.0):
        self.chd, self.oracle, self.mode = chd, oracle, mode
        wc = self.wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], N, S)
        self.N, self.S, self.C, self.step_len = N, S, wc.cells, step
        self.og = make_grid(wc.offx, wc.offz, wc.w, wc.h, wc.cols, wc.rows, wc.server_cols, wc.server_rows)
        self.x, self.z = chd.synth.entities(wc)
        self.idx = (np.arange(S, dtype=np.int64) * max(N // S, 1)) % N
        self.r = np.full(S, wc.radius)
        rng = np.random.default_rng(5)
        self.gid = rng.choice(ID_SPACE, N, replace=False).astype(np.uint32)
        self.ids = (rng.choice((1 << 31) - 1, N, replace=False) + 1).astype(np.uint32)
        self.e = chd.engine.Engine(wc.cfg(), N, S)
        e = self.e
        e.enable_graphs(graphs)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        if mode == "table":
            e.entity_table_init()
            e.reserve_visible_delta(cap)
            assert (e.spawn_entities(self.ids, self.x, self.z) == chd.capi.EV_OK).all()
        elif mode == "id":
            e.reserve_visible_delta_ids(cap, ID_SPACE)
        else:
            e.reserve_visible_delta(cap)
        _, off, arr, snd, ridx, cmi = chd.synth.update_rings(wc, 0, 0, 33 * MS, 4, S, ring_len=64)
        self.rings = (off, arr, snd, ridx, cmi)
        self.t = 0
        self.prev = None  # oracle state of the last successful delta (None: the empty snapshot)

    def enqueue(self, flags, move=True, bad_ids=False):
        """prefetch, adopt, chd_begin_interest, chd_tick(flags) for the next tick; -> the oracle state of that tick"""
        chd, e = self.chd, self.e
        if self.t and move:
            self.x, self.z = chd.synth.move_entities(self.wc, self.x, self.z, self.t, self.step_len)
        self.t += 1
        t_ns = self.t * 33 * MS
        if self.mode == "index":
            e.prefetch_entities(self.x, self.z)
        batch, keep = chd.engine.make_batch(self.S, sub=np.arange(self.S, dtype=np.uint32),
                                            sphere=(self.x[self.idx].copy(), self.z[self.idx].copy(), self.r))
        e.prefetch_queries(batch, keep)
        e.prefetch_rings(*self.rings)
        e.adopt_prefetched()
        if self.mode == "id":
            e.set_entities(self.x, self.z)
            gid = self.gid.copy()
            if bad_ids:  # one id on two in-world entities
                gid[1] = gid[0]
            e.set_entity_ids(gid)
        elif self.mode == "table" and self.t > 1 and move:
            e.move_entities(self.ids, self.x, self.z)
        assert chd.L.chd_begin_interest(e.h, None, t_ns, 1) == 0, e.L.chd_last_error(e.h)
        assert chd.L.chd_tick(e.h, None, t_ns, flags, None) == 0, e.L.chd_last_error(e.h)
        p = self.oracle.sphere_pairs(self.og, self.x, self.z, self.x[self.idx], self.z[self.idx], self.r)
        assert (p["status"] == 0).all()
        return (_cells(self.oracle, self.og, self.x, self.z), p["pair_off"], (p["pair_cell"].astype(np.int64) - S0).astype(np.uint32))

    def want(self, now):
        """the oracle's delta from the last successful one to `now`, in this mode's entity names"""
        if self.mode == "id":
            by_id = np.full(ID_SPACE, self.C, np.uint32)
            by_id[self.gid] = now[0]
            now = (by_id, now[1], now[2])
        prev = self.prev if self.prev is not None else (np.zeros(0, np.uint32), np.zeros(1, np.uint64), np.zeros(0, np.uint32))
        w = self.oracle.visible_delta(self.C, prev, now)
        if self.mode == "table":
            w = (w[0], self.ids[w[1]], w[2], self.ids[w[3]])
        return w, now

    def check(self, got, now, t):
        w, state = self.want(now)
        if self.mode == "id":
            for (go, ge), (wo, we), name in (((got[0], got[1]), (w[0], w[1]), "entered"), ((got[2], got[3]), (w[2], w[3]), "left")):
                np.testing.assert_array_equal(_keys(go, ge, self.S), _keys(wo, we, self.S), err_msg="tick %d %s" % (t, name))
        else:
            for name, u, v in zip(("enter_off", "enter", "leave_off", "leave"), got, w):
                np.testing.assert_array_equal(u, v, err_msg="tick %d %s" % (t, name))
        self.prev = state
        return w

    def close(self):
        self.e.close()


def _fetch_async(chd, w, ds):
    r = chd.capi.ResultBuffers()
    return chd.L.chd_fetch_results_async_delta(w.e.h, C.byref(r), C.byref(ds.b), chd.capi.ptr(ds.hdr))


def _wait(chd, w):
    s, c = chd.capi.TickSummary(), chd.capi.DeltaCounts()
    st = chd.L.chd_fetch_wait_delta(w.e.h, C.byref(s), C.byref(c))
    return st, s, c


def _pipelined(chd, w, flags_of, ticks, sets, move_of=lambda k: True):
    """The e2e loop: enqueue tick k, fetch it, then wait for tick k-1 (two fetches outstanding, two buffer sets) and check it.
    flags_of(k): tick k's flags.  -> per tick (counts, lists or None)"""
    out = []
    pending = []  # (k, state, had delta)
    for k in range(ticks + 1):
        if k < ticks:
            fl = flags_of(k)
            sets[k % 2].reset()
            now = w.enqueue(fl, move=move_of(k))
            assert _fetch_async(chd, w, sets[k % 2]) == 0, w.e.L.chd_last_error(w.e.h)
            pending.append((k, now, bool(fl & chd.capi.TICK_VISIBLE_DELTA)))
        if k == 0:
            continue
        j, now, had = pending.pop(0)
        st, s, c = _wait(chd, w)
        assert st == 0, w.e.L.chd_last_error(w.e.h)
        ds = sets[j % 2]
        if not had:
            assert (c.deltas, c.n_entered, c.n_left, c.n_slots) == (0, 0, 0, 0)
            assert ds.untouched()
            out.append((c, None))
            continue
        assert c.deltas == 1 and c.n_slots == w.S
        got = ds.lists(c)
        want = w.check(got, now, j)
        assert (c.n_entered, c.n_left) == (len(want[1]), len(want[3]))
        out.append((c, got))
    return out


ALL_DELTA = 7 | 8 | 16  # TICK_ALL | TICK_EARLY_RESULTS | TICK_VISIBLE_DELTA


# ------------------------------------------------------------------------------------------------------------ 1. the pipelined loop
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "direct"])
@pytest.mark.parametrize("mode", ["index", "id", "table"])
def test_pipelined_loop_every_tick_exact(chd, oracle, mode, graphs):
    with closing(World(chd, oracle, mode, 30_000, 3_000, graphs)) as w:
        sets = [DeltaSet(chd, w.S + 1, 1 << 22), DeltaSet(chd, w.S + 1, 1 << 22)]
        out = _pipelined(chd, w, lambda k: ALL_DELTA, 9, sets)
        assert all(c.n_entered > 0 and c.n_left > 0 for c, _ in out[1:])


# ------------------------------------------------------------------------------------------------------- 2. ordering under load
def test_next_delta_enqueued_right_after_the_fetch_does_not_corrupt_it(chd, oracle):
    """Large lists (every entity moves up to 600 per axis), tick k+1 and its delta enqueued right after fetch_async_delta(k), two
    fetches outstanding: the delta guard alone keeps tick k's snapshot intact."""
    with closing(World(chd, oracle, "index", 100_000, 20_000, step=600.0)) as w:
        sets = [DeltaSet(chd, w.S + 1, 1 << 24), DeltaSet(chd, w.S + 1, 1 << 24)]
        out = _pipelined(chd, w, lambda k: ALL_DELTA, 8, sets)
        assert min(c.n_entered + c.n_left for c, _ in out[1:]) > 1_000_000


# ---------------------------------------------------------------------------------------------------- 3. sizes where the copy loops
def test_copy_loops_lists_and_offsets_beyond_one_pass(chd, oracle):
    """150 K slots (their offsets need more than one pass of the copy grid), lists up to millions of entries, destinations one
    element past 16-byte alignment, a tick without movement (empty lists) and list lengths that are not multiples of 4."""
    with closing(World(chd, oracle, "index", 3_000, 150_000)) as w:
        assert 2 * (w.S + 1) > chd.copy_pass_words, (w.S, chd.copy_pass_words)
        sets = [DeltaSet(chd, w.S + 1, 1 << 22, shift=1), DeltaSet(chd, w.S + 1, 1 << 22, shift=1)]
        out = _pipelined(chd, w, lambda k: ALL_DELTA, 5, sets, move_of=lambda k: k != 3)
        n = [(c.n_entered, c.n_left) for c, _ in out]
        assert n[0][0] > chd.copy_pass_words, (n, chd.copy_pass_words)
        assert n[3] == (0, 0), n  # nothing moved, the queries are the same: empty lists
        assert any(v % 4 for pair in n for v in pair), n


# ------------------------------------------------------------------------------------------------------- 4. ticks without a delta
def test_ticks_without_a_delta_report_none_and_the_next_covers_both(chd, oracle):
    with closing(World(chd, oracle, "index", 30_000, 3_000)) as w:
        sets = [DeltaSet(chd, w.S + 1, 1 << 22), DeltaSet(chd, w.S + 1, 1 << 22)]
        # the oracle's prev moves only on delta ticks, so each delta is checked against the state two ticks back
        out = _pipelined(chd, w, lambda k: ALL_DELTA if k % 2 == 0 else 7 | 8, 8, sets)
        assert [c.deltas for c, _ in out] == [1, 0] * 4


def test_two_standalone_deltas_between_fetches_report_two_and_the_second_lists(chd, oracle):
    L = chd.L
    with closing(World(chd, oracle, "index", 30_000, 3_000)) as w:
        e = w.e
        ds = DeltaSet(chd, w.S + 1, 1 << 22)
        w.prev = w.enqueue(7 | 8)  # a two-stream tick without the flag
        e.visible_delta()  # delta 1: everything enters (never fetched: lost)
        now = w.enqueue(7 | 8)
        e.visible_delta()  # delta 2: tick 1 -> tick 2
        s, c = chd.capi.TickSummary(), chd.capi.DeltaCounts()
        # the sync form after a two-stream tick (the early read-back path)
        assert L.chd_fetch_results_delta(e.h, C.byref(chd.capi.ResultBuffers()), C.byref(ds.b), C.byref(s), C.byref(c)) == 0
        assert c.deltas == 2 and c.n_slots == w.S
        got = ds.lists(c)
        assert len(got[1]) and len(got[3])
        w.check(got, now, 1)
        for u, v in zip(got, e.get_visible_delta()):
            np.testing.assert_array_equal(u, v)
        # a fetch right after: nothing new
        ds.reset()
        assert L.chd_fetch_results_delta(e.h, C.byref(chd.capi.ResultBuffers()), C.byref(ds.b), C.byref(s), C.byref(c)) == 0
        assert c.deltas == 0 and ds.untouched()


def test_standalone_delta_on_a_single_stream_tick_sync_form(chd, oracle):
    L = chd.L
    with closing(World(chd, oracle, "index", 30_000, 3_000)) as w:
        e = w.e
        ds = DeltaSet(chd, w.S + 1, 1 << 22)
        for t in range(3):
            if t:
                w.x, w.z = chd.synth.move_entities(w.wc, w.x, w.z, t, 150.0)
            e.set_entities(w.x, w.z)
            batch, keep = chd.engine.make_batch(w.S, sub=np.arange(w.S, dtype=np.uint32), sphere=(w.x[w.idx].copy(), w.z[w.idx].copy(), w.r))
            e.update_interest(batch, (t + 1) * 33 * MS)
            e.tick(None, (t + 1) * 33 * MS, chd.capi.TICK_BUILD, want_summary=False)  # one stream: no early read-back
            e.visible_delta()
            p = oracle.sphere_pairs(w.og, w.x, w.z, w.x[w.idx], w.z[w.idx], w.r)
            now = (_cells(oracle, w.og, w.x, w.z), p["pair_off"], (p["pair_cell"].astype(np.int64) - S0).astype(np.uint32))
            ds.reset()
            s, c = chd.capi.TickSummary(), chd.capi.DeltaCounts()
            assert L.chd_fetch_results_delta(e.h, C.byref(chd.capi.ResultBuffers()), C.byref(ds.b), C.byref(s), C.byref(c)) == 0
            assert c.deltas == 1 and c.n_slots == w.S
            w.check(ds.lists(c), now, t)


# -------------------------------------------------------------------------------------------------------------------- 5. overflow
@pytest.mark.parametrize("kind", ["delta", "delta_ids"])
def test_overflow_reports_required_sizes_and_the_next_fetch_catches_up(chd, oracle, kind):
    """CHD_OVF_DELTA: a reserve of 16 entries, too small for the first delta (everything enters).  CHD_OVF_DELTA_IDS: one id on two
    in-world entities in the first tick.  The wait returns CHD_ERR_CAPACITY with the required sizes and writes no delta buffer; the
    next fetched delta (after a larger reserve) covers everything since the empty snapshot."""
    mode = "index" if kind == "delta" else "id"
    with closing(World(chd, oracle, mode, 30_000, 3_000, cap=16 if kind == "delta" else 1 << 22)) as w:
        e = w.e
        sets = [DeltaSet(chd, w.S + 1, 1 << 22), DeltaSet(chd, w.S + 1, 1 << 22)]
        ds = sets[0]
        ds.reset()
        now = w.enqueue(ALL_DELTA, bad_ids=(kind == "delta_ids"))
        assert _fetch_async(chd, w, ds) == 0
        st, s, c = _wait(chd, w)
        assert st == chd.capi.ERR_CAPACITY
        want_bit = chd.capi.OVF_DELTA if kind == "delta" else chd.capi.OVF_DELTA_IDS
        assert s.overflow & want_bit and c.deltas == 1
        assert ds.untouched()
        if kind == "delta":
            w_, _ = w.want(now)  # the required sizes (the snapshot did not advance)
            assert (c.n_entered, c.n_left) == (len(w_[1]), len(w_[3])) and c.n_entered > 16
            e.reserve_visible_delta(1 << 22)
        # the next delta covers everything since the last successful one
        out = _pipelined(chd, w, lambda k: ALL_DELTA, 2, sets)
        assert out[0][0].n_entered > 0


# ------------------------------------------------------------------------------------------------------------------ 6. caller caps
def test_caller_caps_too_small_async_truncates_sync_refuses(chd, oracle):
    L = chd.L
    with closing(World(chd, oracle, "index", 30_000, 3_000)) as w:
        e = w.e
        small = DeltaSet(chd, w.S + 1, 1000)
        now = w.enqueue(ALL_DELTA)
        assert _fetch_async(chd, w, small) == 0
        st, s, c = _wait(chd, w)
        assert st == chd.capi.ERR_CAPACITY and s.overflow == 0 and c.deltas == 1 and c.n_entered > 1000
        want = w.check(e.get_visible_delta(), now, 0)
        np.testing.assert_array_equal(small.en.numpy()[:1000].view(np.uint32), want[1][:1000])
        np.testing.assert_array_equal(small.eo.numpy().view(np.uint64), want[0])
        # sync form, slot_cap or entity_cap too small: nothing written
        for ds in (DeltaSet(chd, w.S, 1 << 22), DeltaSet(chd, w.S + 1, 10)):
            w.enqueue(ALL_DELTA)
            assert L.chd_fetch_results_delta(e.h, C.byref(chd.capi.ResultBuffers()), C.byref(ds.b), C.byref(s), C.byref(c)) == chd.capi.ERR_CAPACITY
            assert ds.untouched()


# ----------------------------------------------------------------------------------------------------- 7. chd_tick_sharded at world 1
@pytest.mark.parametrize("table", [False, True], ids=["ids", "table_on_slab"])
def test_tick_sharded_at_world_one(chd, table):
    L = chd.L
    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 20_000, 1_000)
    N, S = wc.n_entities, wc.n_subscribers
    x, z = chd.synth.entities(wc)
    idx = (np.arange(S, dtype=np.int64) * (N // S)) % N
    from channeld_b200 import sharding

    e = chd.engine.Engine(wc.cfg(), 2 * N + 16, S, max_visible=1 << 25)
    try:
        e.comm_init(chd.engine.Engine.comm_unique_id(), 0, 1, sharding.halo_columns(1000.0, wc.w), N)
        ids = (np.arange(N, dtype=np.uint32) * 7 + 1) % ID_SPACE
        if table:
            e.entity_table_init()
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.reserve_visible_delta_ids(1 << 22, ID_SPACE)
        if table:
            assert (e.spawn_entities(ids, x, z) == chd.capi.EV_OK).all()
        ds = DeltaSet(chd, S + 1, 1 << 22)
        for t in range(4):
            if t:
                x, z = chd.synth.move_entities(wc, x, z, t, 300.0)
                if table:
                    e.move_entities(ids, x, z)
            if not table:
                e.set_entities(x, z)
                e.set_entity_ids(ids)
            batch, keep = chd.engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(x[idx].copy(), z[idx].copy(), np.full(S, 1000.0)))
            e.tick_sharded(batch, (t + 1) * 33 * MS, 1 | 2 | 16, want_summary=False)
            ds.reset()
            s, c = chd.capi.TickSummary(), chd.capi.DeltaCounts()
            assert L.chd_fetch_results_delta(e.h, C.byref(chd.capi.ResultBuffers()), C.byref(ds.b), C.byref(s), C.byref(c)) == 0, \
                e.L.chd_last_error(e.h)
            assert c.deltas == 1 and c.n_slots == S and c.n_entered > 0
            for u, v in zip(ds.lists(c), e.get_visible_delta()):  # what chd_get_visible_delta returns right after the delta
                np.testing.assert_array_equal(u, v)
        assert L.chd_comm_destroy(e.h) == chd.capi.OK
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------ 8. argument errors
def test_argument_errors(chd, oracle):
    L = chd.L
    wc = chd.synth.scaled(chd.synth.CONFIGS["benchmark"], 2_000, 100)
    with closing(chd.engine.Engine(wc.cfg(), 2_000, 100)) as e:
        ds = DeltaSet(chd, 101, 1 << 16)
        r, s, c = chd.capi.ResultBuffers(), chd.capi.TickSummary(), chd.capi.DeltaCounts()
        e.set_subscribers(np.arange(1, 101, dtype=np.uint32))
        x, z = chd.synth.entities(wc)
        e.set_entities(x, z)
        batch, keep = chd.engine.make_batch(100, sub=np.arange(100, dtype=np.uint32), sphere=(x[:100].copy(), z[:100].copy(), np.full(100, 50.0)))
        e.tick(batch, 33 * MS, 7 | 8, want_summary=False)
        # no reserve yet: CHD_ERR_STATE for delta buffers, both forms
        assert L.chd_fetch_results_async_delta(e.h, C.byref(r), C.byref(ds.b), chd.capi.ptr(ds.hdr)) == chd.capi.ERR_STATE
        assert L.chd_fetch_results_delta(e.h, C.byref(r), C.byref(ds.b), C.byref(s), C.byref(c)) == chd.capi.ERR_STATE
        e.reserve_visible_delta(1 << 16)
        e.tick(batch, 66 * MS, ALL_DELTA, want_summary=False)
        # pageable (not pinned) delta buffers: CHD_ERR_INVALID
        host = np.zeros(1 << 16, np.uint32)
        bad = chd.capi.DeltaBuffers()
        bad.enter_entity, bad.entity_cap = chd.capi.ptr(host), 1 << 16
        assert L.chd_fetch_results_async_delta(e.h, C.byref(r), C.byref(bad), chd.capi.ptr(ds.hdr)) == chd.capi.ERR_INVALID
        # delta == NULL: the plain fetch; its wait reports no delta
        assert L.chd_fetch_results_async_delta(e.h, C.byref(r), None, chd.capi.ptr(ds.hdr)) == 0
        assert L.chd_fetch_wait_delta(e.h, C.byref(s), C.byref(c)) == 0
        assert c.deltas == 0
