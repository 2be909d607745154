"""Byte-carrying device rings (include/chd_gpu_ring_bytes.h): each update's serialized updateMsg kept in the ring beside its entry,
evicted, slid and dropped with it, and read in place by chd_assemble_payloads / chd_frame_packets.

  ring parity   the world of tests/test_gpu_rings_scale.py (100 K subscribers, floods of 150-400 updates in hot cells, 8
                irregular ticks) on grids a (225 cells), b (300) and e (65 536) with entry slabs of 513, 620 and 1024 and a byte
                slab that never drops: every tick the rings equal the oracle's and an engine without bytes fed the same updates,
                the due lists of the two engines are equal, and every live entry's bytes are those of its (cell, msgIndex)
  payloads     every class entry is _wire.class_entry of the bytes of the ring entries the oracle's window selected (the full
                data for FULL sends); every connection's frames match the restated flush, with snappy and raw connections and
                full data messages at the drop limit and one byte below it; each decision's entry, found by its identity
                (connection, channel, kind, window_hi, last_message_index), equals that of a host-owned-ring engine given the same
                rings and bytes; through chd_fanout_tick and chd_tick(TICK_ALL) with graphs on and off
  capacity      a byte slab small enough to drop: rings, msgIndex and bytes equal tests/_ring_bytes.py's restatement, including a
                byte slide by fewer than 32 bytes, CHD_OVF_RING exactly on the ticks that dropped, and an update longer than the
                slab refused with nothing changed
  rules         every clause of mode rule 14 and rules 12 / 13 for the new calls: refused, nothing changed, no launch
Run on an H100:  python -m pytest tests/test_ring_bytes_gpu.py -m gpu
"""
import ctypes as C

import numpy as np
import pytest

from tests._ring_bytes import ByteRing, entry_bytes, msg_indices, update_bytes
from tests.test_gpu_payload_scale import DROP_ENTRY, MP_DROP, Payload, _value_len_for_mp, check_frames, restate_frames
from tests.test_gpu_rings_scale import (N_TICKS, S0, _assert_rings, _csr, _due_from, _engine, _Reference, _status, _World, chd)  # noqa: F401

pytestmark = pytest.mark.gpu

MS = 1_000_000
MAX_LEN = 23  # longest update the tests give (tests/_ring_bytes.py)


def _append_bytes(chd, e, upd_off, arrival, sender, msg_before):
    """chd_rings_append_bytes of updates CSR by cell, each carrying entry_bytes(cell, its msgIndex) -> status"""
    cell, idx = msg_indices(upd_off, msg_before)
    boff, data = update_bytes(cell, idx, MAX_LEN)
    p = chd.capi.ptr
    upd_off = np.ascontiguousarray(upd_off, np.uint32)
    arrival, sender = np.ascontiguousarray(arrival, np.int64), np.ascontiguousarray(sender, np.uint32)
    n = len(boff) - 1
    return e.L.chd_rings_append_bytes(e.h, p(upd_off), n, p(arrival) if n else None, p(sender) if n else None, p(boff),
                                      p(data) if len(data) else None)


def _want_bytes(rings, n_cells):
    cell = np.repeat(np.arange(n_cells), np.diff(rings["off"].astype(np.int64)))
    parts = [entry_bytes(c, i, MAX_LEN) for c, i in zip(cell.tolist(), rings["index"].tolist())]
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in parts])
    return off, b"".join(parts)


def _assert_bytes(e, rings):
    off, data = e.get_ring_bytes()
    w_off, w_data = _want_bytes(rings, e.n_cells)
    np.testing.assert_array_equal(off, w_off)
    assert data.tobytes() == w_data


def _entries_by_decision(conn, e, due, cls_off, blob):
    """-> (sorted list of ((connection, channel, kind, window_hi, last_message_index), class entry bytes), due["sub"])"""
    cls_of = e.due_classes(len(due["sub"]))[0].astype(np.int64)
    out = []
    for i in range(len(cls_of)):
        k = cls_of[i]
        key = (int(conn[due["sub"][i]]), int(due["channel_id"][i]), int(due["kind"][i]), int(due["window_hi"][i]), int(due["last_message_index"][i]))
        out.append((key, blob[int(cls_off[k]):int(cls_off[k + 1])].tobytes()))
    return sorted(out), due["sub"]


def _summary_overflow(chd, e):
    s = chd.capi.TickSummary()
    e.L.chd_summary(e.h, C.byref(s))
    return int(s.overflow)


@pytest.mark.parametrize("grid,cap", [("a", 513), ("b", 620), ("e", 1024)], ids=["a-cap513", "b-cap620", "e-cap1024"])
def test_ring_parity(chd, oracle, grid, cap):
    w = _World(oracle, grid, 7100 + cap + ord(grid))
    ref = _Reference(oracle, w, cap)
    e = _engine(chd, w, cap)
    e.rings_reserve_bytes(cap * (MAX_LEN + 1))  # never drops: a full entry slab of the longest updates fits
    plain = _engine(chd, w, cap)
    hot = np.nonzero(w.hot)[0]
    rest = {int(c): ByteRing(cap, cap * (MAX_LEN + 1)) for c in hot}
    msg_before = np.zeros(w.C, np.uint64)
    for tick in range(N_TICKS):
        t, cx, cz, rad = w.next_tick(tick)
        want = oracle.sphere_pairs(w.og, np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]), cx, cz, rad)
        batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(cx, cz, rad))
        for x in (e, plain):
            x.update_interest(batch, t)
            x.summary()
        r = ref.tick(tick, t, want)
        e._ck(_append_bytes(chd, e, r["upd_off"], r["u_arr"], r["u_snd"], msg_before))
        plain.rings_append(r["upd_off"], r["u_arr"], r["u_snd"])
        got = e.get_rings()
        _assert_rings(got, r["rings"])
        _assert_rings(got, plain.get_rings())
        _assert_bytes(e, got)
        # the restatement of the hot cells (every other cell holds a few entries at its slab starts)
        uo = r["upd_off"].astype(np.int64)
        cell_idx, idx = msg_indices(r["upd_off"], msg_before)
        for c, br in rest.items():
            for k in range(uo[c], uo[c + 1]):
                assert br.append(r["u_arr"][k], r["u_snd"][k], entry_bytes(c, idx[k], MAX_LEN), r["rings"]["max_interval_ms"][c]) == 0
            go = got["off"].astype(np.int64)
            assert [x[2] for x in br.ents] == got["index"][go[c]:go[c + 1]].tolist()
        msg_before = got["msg_index"].copy()
        for x in (e, plain):
            x.fanout_tick(t)
        s, sp = e.summary(), plain.summary()
        assert s.overflow == 0 and sp.overflow == 0 and s.n_due == sp.n_due == len(r["due"])
        np.testing.assert_array_equal(_due_from(w.conn, e.get_due(s.n_due)), r["due"])
        np.testing.assert_array_equal(_due_from(w.conn, plain.get_due(sp.n_due)), r["due"])
    e.close()
    plain.close()
    rs = list(rest.values())
    assert sum(x.evictions for x in rs) > 0 and sum(x.slides for x in rs) > 0 and sum(len(x.byte_slides) for x in rs) > 0
    assert sum(x.drops for x in rs) == 0


class _Selecting(_Reference):
    """_Reference whose oracle tick also reports which ring entries each send merged (tick_data_ex)"""

    def _tick_data(self, t, cap):
        sends, soff, lo, sk, sel_off, sel_pos = self.chans.tick_data_ex(t, cap, 1 << 26)
        self.sel = dict(sends=sends, soff=soff, sel_off=sel_off, sel_pos=sel_pos)
        return sends, np.repeat(np.arange(self.w.C), np.diff(soff.astype(np.int64)))


def _payload_world(chd, oracle, graphs, seed):
    w = _World(oracle, "b", seed, n_sub=40_000)
    return w, _engine(chd, w, 1024, graphs=graphs)


@pytest.mark.parametrize("mode", ["fanout", "tick-graphs", "tick-nographs"])
def test_payloads(chd, oracle, mode):
    """chd_assemble_payloads / chd_frame_packets on byte-carrying rings: every class entry is _wire.class_entry of the
    concatenated bytes of the ring entries the oracle's window selected (the full data for FULL sends), every connection's frames
    are connection.go's flush as tests/test_gpu_payload_scale.py restates it (full data messages at the drop limit dropped, just
    below it kept), and each decision's entry equals that of a host-owned-ring engine given the same rings and bytes."""
    from tests import _wire as W

    capi = chd.capi
    graphs = mode != "tick-nographs"
    cap = 1024
    w, e = _payload_world(chd, oracle, graphs, 9300 + len(mode))
    e.rings_reserve_bytes(cap * (MAX_LEN + 1))
    ref = _Selecting(oracle, w, cap, rings_first=mode != "fanout")
    h = chd.engine.Engine(chd.engine.grid_cfg(*w.g), 1, w.S, max_pairs=1 << 21, max_due=1 << 23, max_ring_entries=w.C * cap,
                          max_window_cells=w.S * 48 + 65536)
    h.enable_graphs(graphs)
    h.set_entities(np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]))
    h.set_subscribers(w.conn)
    h.build()
    pe, ph = Payload(chd, e, w.S), Payload(chd, h, w.S)
    rng = np.random.default_rng(31)
    compression = (np.arange(w.S) % 2).astype(np.uint8)
    msg_before = np.zeros(w.C, np.uint64)
    n_update_cls = n_dropped = n_below = 0
    for tick in range(N_TICKS):
        t, cx, cz, rad = w.next_tick(tick)
        want = oracle.sphere_pairs(w.og, np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]), cx, cz, rad)
        batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(cx, cz, rad))
        if mode == "fanout":
            e.update_interest(batch, t)
            e.summary()
        r = ref.tick(tick, t, want)
        e._ck(_append_bytes(chd, e, r["upd_off"], r["u_arr"], r["u_snd"], msg_before))
        rings = e.get_rings()
        _assert_rings(rings, r["rings"])
        msg_before = rings["msg_index"].copy()
        eoff, eb = e.get_ring_bytes()
        f_len = (rng.random(w.C) ** 3 * 400).astype(np.int64)
        f_len[tick % w.C] = 30000  # a large full data message
        at = np.arange(w.C) % 10 == tick % 10  # MessagePacks at the drop limit (dropped) and one byte below it (kept)
        below = np.arange(w.C) % 10 == (tick + 5) % 10
        f_len[at] = [_value_len_for_mp(MP_DROP, S0 + c) for c in np.nonzero(at)[0]]
        f_len[below] = [_value_len_for_mp(MP_DROP - 1, S0 + c) for c in np.nonzero(below)[0]]
        foff = np.concatenate([[0], np.cumsum(f_len)]).astype(np.uint64)
        fb = np.frombuffer(rng.bytes(int(foff[-1])), np.uint8)
        pe.set_bytes(np.zeros(1, np.uint64), np.zeros(0, np.uint8), foff, fb)
        h.set_rings(rings["off"], rings["arrival"], rings["sender"], rings["index"], rings["msg_index"])
        ph.set_bytes(eoff, eb, foff, fb)
        if mode == "fanout":
            e.fanout_tick(t)
            h.update_interest(batch, t)
            h.fanout_tick(t)
        else:
            e.tick(batch, t, capi.TICK_ALL, want_summary=False)
            h.tick(batch, t, capi.TICK_ALL, want_summary=False)
        n_cls, cls_off, blob = pe.assemble()
        n_cls_h, cls_off_h, blob_h = ph.assemble()
        frames, frames_h = pe.frame(compression), ph.frame(compression)
        s, sh = e.summary(), h.summary()
        assert s.overflow == 0 and sh.overflow == 0 and s.n_due == sh.n_due == len(r["due"])
        due = e.get_due(s.n_due)
        np.testing.assert_array_equal(_due_from(w.conn, due), r["due"])
        np.testing.assert_array_equal(_due_from(w.conn, h.get_due(sh.n_due)), r["due"])
        # the due lists are unordered: each decision's class entry, by its identity
        assert n_cls == n_cls_h
        entries = [_entries_by_decision(w.conn, x, d, co, b) for x, d, co, b in ((e, due, cls_off, blob), (h, h.get_due(sh.n_due), cls_off_h, blob_h))]
        assert entries[0][0] == entries[1][0]
        check_frames(restate_frames(entries[1][1], np.arange(sh.n_due), h.due_classes(sh.n_due)[0].astype(np.int64), np.diff(cls_off_h.astype(np.int64)), w.S,
                                    compression), cls_off_h, blob_h, frames_h, w.S, compression)
        cls_of, cls_rep, cls_cnt = e.due_classes(s.n_due)
        restated = restate_frames(due["sub"], np.arange(s.n_due), cls_of.astype(np.int64), np.diff(cls_off.astype(np.int64)), w.S, compression)
        check_frames(restated, cls_off, blob, frames, w.S, compression)
        # every class entry from the oracle's selection for its representative decision
        sel = ref.sel
        s_cell = np.repeat(np.arange(w.C), np.diff(sel["soff"].astype(np.int64)))
        sends = sel["sends"]
        j_of = {(int(sends["conn_id"][j]), int(s_cell[j]) + S0, int(sends["kind"][j]), int(sends["window_hi"][j]), int(sends["last_message_index"][j])): j
                for j in range(len(sends))}
        assert len(j_of) == len(sends)
        ro = rings["off"].astype(np.int64)
        for k, i in enumerate(cls_rep.tolist()):
            c = int(due["channel_id"][i]) - S0
            j = j_of[(int(w.conn[due["sub"][i]]), c + S0, int(due["kind"][i]), int(due["window_hi"][i]), int(due["last_message_index"][i]))]
            if due["kind"][i] == 0:
                value = fb[int(foff[c]):int(foff[c + 1])].tobytes()
            else:
                pos = sel["sel_pos"][int(sel["sel_off"][j]):int(sel["sel_off"][j + 1])]
                value = b"".join(entry_bytes(c, int(rings["index"][ro[c] + q]), MAX_LEN) for q in pos.tolist())
            assert blob[int(cls_off[k]):int(cls_off[k + 1])].tobytes() == W.class_entry(c + S0, value), (tick, k)
        cls_len = np.diff(cls_off.astype(np.int64))
        n_update_cls += int((due["kind"][cls_rep] == 1).sum())
        n_dropped += frames[4]
        n_below += int((cls_len == DROP_ENTRY - 1).sum())
    assert n_update_cls > 1000 and n_dropped > 0 and n_below > 0
    e.close()
    h.close()


def test_byte_capacity(chd, oracle):
    """A byte slab of 1000 bytes on 1024-entry slabs, no subscribers (maxFanOutIntervalMs 0): the rings, msgIndex and bytes equal
    the restatement every tick, CHD_OVF_RING is raised exactly on the ticks that dropped, and an update longer than the slab is
    refused with nothing changed."""
    capi = chd.capi
    cap, bcap = 1024, 1000
    w = _World(oracle, "b", 51, n_sub=16, n_hot=0)
    e = chd.engine.Engine(chd.engine.grid_cfg(*w.g), 1, w.S, max_ring_entries=w.C * cap)
    e.set_entities(np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]))
    e.set_subscribers(w.conn)
    e.build()
    e.rings_init(cap)
    e.rings_reserve_bytes(bcap)
    rest = [ByteRing(cap, bcap) for _ in range(w.C)]
    rng = np.random.default_rng(52)
    t = 0
    dropped_ticks = []
    for tick in range(6):
        t += 100 * MS
        n_cell = rng.integers(0, 11, w.C)
        n_cell[0] = [530, 1, 0, 0, 0, 0][tick]  # cell 0: 530 one-byte updates, then 480 bytes: a slide by 18 bytes
        n_cell[1] = 3 if tick == 2 else 0       # cell 1: 40 + 40 + 30 in a 1000-byte slab does not drop; 3 x 400 does
        n = int(n_cell.sum())
        upd_off = _csr(n_cell)
        arr = (t + np.arange(n)).astype(np.int64)
        snd = rng.integers(1, 100, n).astype(np.uint32)
        lens = rng.integers(0, 21, n)  # (other cells stay below 1000 live bytes)
        lens[upd_off[0]:upd_off[1]] = 480 if tick == 1 else 1
        lens[upd_off[1]:upd_off[2]] = 400
        parts = [bytes(rng.integers(0, 256, int(L), dtype=np.uint8)) for L in lens]
        boff = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        data = np.frombuffer(b"".join(parts), np.uint8)
        drops = 0
        for c in range(w.C):
            for k in range(int(upd_off[c]), int(upd_off[c + 1])):
                drops += rest[c].append(arr[k], snd[k], parts[k], 0)
        if drops:
            dropped_ticks.append(tick)
        e.rings_append_bytes(upd_off, arr, snd, boff, data)
        assert bool(_summary_overflow(chd, e) & capi.OVF_RING) == (drops > 0), tick
        got = e.get_rings()
        go = got["off"].astype(np.int64)
        for c in range(w.C):
            ents = rest[c].ents
            assert got["index"][go[c]:go[c + 1]].tolist() == [x[2] for x in ents], c
            assert got["arrival"][go[c]:go[c + 1]].tolist() == [x[0] for x in ents], c
            assert got["sender"][go[c]:go[c + 1]].tolist() == [x[1] for x in ents], c
        np.testing.assert_array_equal(got["msg_index"], [r.mi for r in rest])
        off, blob = e.get_ring_bytes()
        want = b"".join(x[3] for r in rest for x in r.ents)
        assert blob.tobytes() == want
        np.testing.assert_array_equal(np.diff(off.astype(np.int64)), [len(x[3]) for r in rest for x in r.ents])
    assert 18 in rest[0].byte_slides and rest[1].drops == 1 and dropped_ticks == [2]
    # an update longer than the slab: CHD_ERR_INVALID, nothing appended, no launch
    before, before_bytes, launches = e.get_rings(), e.get_ring_bytes(), e.launch_count()
    n_cell = np.zeros(w.C, np.int64)
    n_cell[[3, 4]] = 1
    boff = np.array([0, 10, 10 + bcap + 1], np.uint64)
    data = np.zeros(int(boff[-1]), np.uint8)
    p = capi.ptr
    uo = _csr(n_cell)
    arr, snd = np.full(2, t, np.int64), np.ones(2, np.uint32)
    assert e.L.chd_rings_append_bytes(e.h, p(uo), 2, p(arr), p(snd), p(boff), p(data)) == capi.ERR_INVALID
    assert e.launch_count() == launches
    after = e.get_rings()
    for k in before:
        np.testing.assert_array_equal(after[k], before[k])
    assert e.get_ring_bytes()[1].tobytes() == before_bytes[1].tobytes()
    e.close()


def test_rules(chd, oracle):
    """Mode rule 14 and rules 12 / 13 for the new calls: each refused call returns its status, launches nothing and changes
    nothing."""
    capi = chd.capi
    p = capi.ptr
    cap = 1024
    w = _World(oracle, "b", 61, n_sub=2000, n_hot=0)
    w.hot[:] = False

    def fresh(init=True):
        e = chd.engine.Engine(chd.engine.grid_cfg(*w.g), 1, w.S, max_ring_entries=w.C * cap, max_pairs=1 << 20, max_due=1 << 20,
                              max_window_cells=w.S * 48 + 65536)
        e.set_entities(np.array([w.g[0] + 1.0]), np.array([w.g[1] + 1.0]))
        e.set_subscribers(w.conn)
        e.build()
        if init:
            e.rings_init(cap)
        return e

    def refused(e, st, call):
        n = e.launch_count()
        assert call() == st
        assert e.launch_count() == n

    n_cell = np.full(w.C, 2)
    upd_off = _csr(n_cell)
    arr = np.full(int(upd_off[-1]), 5 * MS, np.int64)
    snd = np.full(int(upd_off[-1]), 7, np.uint32)
    zero = np.zeros(w.C, np.uint64)
    # the reserve: after chd_rings_init, before any append
    e = fresh(init=False)
    refused(e, capi.ERR_STATE, lambda: e.L.chd_rings_reserve_bytes(e.h, 256))
    e.rings_init(cap)
    refused(e, capi.ERR_INVALID, lambda: e.L.chd_rings_reserve_bytes(e.h, 0))
    e.rings_append(upd_off, arr, snd)
    refused(e, capi.ERR_STATE, lambda: e.L.chd_rings_reserve_bytes(e.h, 256))
    # an engine without the reservation refuses chd_rings_append_bytes
    rings = e.get_rings()
    refused(e, capi.ERR_STATE, lambda: _append_bytes(chd, e, upd_off, arr, snd, rings["msg_index"]))
    _assert_rings(e.get_rings(), rings)
    # ... and chd_assemble_payloads on device rings, as before
    pl = Payload(chd, e, w.S)
    pl.set_bytes(np.zeros(1, np.uint64), np.zeros(0, np.uint8), np.zeros(w.C + 1, np.uint64), np.zeros(0, np.uint8))
    e.fanout_tick(10 * MS)
    e.summary()
    ncls, blen = C.c_uint32(), C.c_uint64()
    refused(e, capi.ERR_STATE, lambda: e.L.chd_assemble_payloads(e.h, C.byref(ncls), None, 0, None, 0, C.byref(blen)))
    refused(e, capi.ERR_STATE, lambda: e.L.chd_get_ring_bytes(e.h, None, None, 0, None))
    e.close()
    # a byte-carrying engine refuses chd_rings_append; a later chd_rings_init keeps the reservation and empties the slabs
    e = fresh()
    e.rings_reserve_bytes(256)
    e.rings_reserve_bytes(512)  # again before any append: accepted
    e._ck(_append_bytes(chd, e, upd_off, arr, snd, zero))
    rings = e.get_rings()
    refused(e, capi.ERR_STATE, lambda: _status(lambda: e.rings_append(upd_off, arr, snd)))
    refused(e, capi.ERR_STATE, lambda: e.L.chd_rings_reserve_bytes(e.h, 512))
    _assert_rings(e.get_rings(), rings)
    _assert_bytes(e, rings)
    # chd_set_payload_bytes with entries: CHD_ERR_INVALID
    eo = np.array([0, 1], np.uint64)
    eb = np.zeros(1, np.uint8)
    fo = np.zeros(w.C + 1, np.uint64)
    refused(e, capi.ERR_INVALID, lambda: e.L.chd_set_payload_bytes(e.h, p(eo), 1, p(eb), p(fo), p(eb), b"t", 8))
    pl = Payload(chd, e, w.S)
    pl.set_bytes(np.zeros(1, np.uint64), np.zeros(0, np.uint8), fo, np.zeros(0, np.uint8))
    # assemble after an append applied since the last fan-out pass: refused; after the fan-out: accepted
    refused(e, capi.ERR_STATE, lambda: e.L.chd_assemble_payloads(e.h, C.byref(ncls), None, 0, None, 0, C.byref(blen)))
    e.fanout_tick(10 * MS)
    e.summary()
    assert e.L.chd_assemble_payloads(e.h, C.byref(ncls), None, 0, None, 0, C.byref(blen)) == capi.OK
    e._ck(_append_bytes(chd, e, upd_off, (arr + 10 * MS).astype(np.int64), snd, rings["msg_index"]))
    refused(e, capi.ERR_STATE, lambda: e.L.chd_assemble_payloads(e.h, C.byref(ncls), None, 0, None, 0, C.byref(blen)))
    rings = e.get_rings()
    e.rings_init(cap)
    empty = e.get_rings()
    assert int(empty["off"][-1]) == 0
    assert e.get_ring_bytes()[1].size == 0
    refused(e, capi.ERR_STATE, lambda: e.L.chd_assemble_payloads(e.h, C.byref(ncls), None, 0, None, 0, C.byref(blen)))
    e._ck(_append_bytes(chd, e, upd_off, arr, snd, zero))  # the reservation survived chd_rings_init
    _assert_bytes(e, e.get_rings())
    # rule 13: the reserve and the append are refused while a chd_begin_interest is pending
    rings = e.get_rings()
    batch, keep = chd.engine.make_batch(w.S, sub=None, sphere=(w.cx, w.cz, w.rad))
    e.begin_interest(batch, 20 * MS, with_fanout=True)
    refused(e, capi.ERR_STATE, lambda: _append_bytes(chd, e, upd_off, arr, snd, rings["msg_index"]))
    refused(e, capi.ERR_STATE, lambda: e.L.chd_rings_reserve_bytes(e.h, 512))
    e.tick(None, 20 * MS, capi.TICK_ALL)
    _assert_rings(e.get_rings(), rings)
    _assert_bytes(e, rings)
    e.close()
    e = fresh()
    e.begin_interest(batch, 20 * MS, with_fanout=False)
    refused(e, capi.ERR_STATE, lambda: e.L.chd_rings_reserve_bytes(e.h, 512))
    e.tick(None, 20 * MS, capi.TICK_ALL)
    e.rings_reserve_bytes(512)
    e.close()
