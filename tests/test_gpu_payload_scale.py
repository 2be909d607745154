"""The byte half of the fan-out (chd_due_classes, chd_assemble_payloads, chd_frame_packets) at scale, against the batched
tickData emulation of the oracle (orc_channels_tick_data_ex) and the protobuf runtime: every decision, class and connection of
six ticks of 100 K moving subscribers.

  case    world                                                what it exercises
  a       the benchmark grid (15 x 15), bench.py's ring          many UPDATE classes, and connections with hundreds of
          generator, radii 50 / 1500 / 2500, graphs on          decisions split over several packets
  e       256 x 256 cells, radii 50 .. 120                       tens of thousands of FULL classes in the first tick
  a-tick  case a driven by chd_tick(TICK_ALL)                    the payload calls run while the tick's visible-list copy
                                                                 may still be pending
Every case asserts that the due list and both frame scans span several 4 096-element tiles, that some connection has at
least 200 decisions in more than one packet, and that messages at the drop limit are dropped; case e also that the class-length
scan spans several tiles and that its site is rebuilt for a larger class count.

Also here: a due list that overflows (CHD_OVF_DUE) holds CHD_DUE_VOID holes; they belong to no class and are never framed.
Run on an H100:  python -m pytest tests/test_gpu_payload_scale.py -m gpu
"""
import ctypes as C
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S0 = 65536
MS = 1_000_000
N_TICKS = 6
SCAN_TILE = 4096                          # chd_scan.cuh: a look-back scan over more elements spans several tiles
PKT_MAX = 0xFFFF                          # connection.go:27
MP_DROP = PKT_MAX - 5                     # connection.go:73-77: a MessagePack of this size or more is dropped
DROP_ENTRY = 1 + 3 + MP_DROP              # the entry holding such a MessagePack: 0x0A, a 3-byte length varint, the MessagePack
SNAPPY_FITS_UP_TO = 56146                 # snappy.MaxEncodedLen(n) = 32 + n + n/6 <= 0xFFFF up to here
HEAVY = 16                                # subscribers whose sphere covers at least 200 cells

GRIDS = {"a": (-15000.0, -15000.0, 2000.0, 2000.0, 15, 15), "e": (-12800.0, -12800.0, 100.0, 100.0, 256, 256)}
RADII = {"a": (50.0, 1500.0, 2500.0), "e": (50.0, 60.0, 80.0, 120.0)}
HEAVY_R = {"a": 30000.0, "e": 1000.0}     # a: the whole 15 x 15 world from its centre; e: about 340 cells


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
    return ns


def _gather(src, start, length, chunk=1 << 24):
    """The concatenation of src[start[k] : start[k] + length[k]] over k (index arrays of about `chunk` entries at a time)."""
    start, length = np.asarray(start, np.int64), np.asarray(length, np.int64)
    end = np.cumsum(length)
    total = int(end[-1]) if len(end) else 0
    cuts = np.concatenate([[0], np.searchsorted(end, np.arange(chunk, total, chunk)) + 1, [len(end)]])
    parts = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        if b > a:
            s, n = start[a:b], length[a:b]
            parts.append(src[np.repeat(s - (np.cumsum(n) - n), n) + np.arange(int(n.sum()))])
    return np.concatenate(parts) if parts else np.zeros(0, src.dtype)


def _snappy_decode(body):
    import pyarrow as pa

    n, shift, i = 0, 0, 0  # uncompressed length varint
    while True:
        b = body[i]
        n |= (b & 0x7F) << shift
        i += 1
        shift += 7
        if not b & 0x80:
            break
    return pa.decompress(bytes(body), decompressed_size=n, codec="snappy", asbytes=True)


def _value_len_for_mp(target, ch):
    """The value length whose MessagePack for channel `ch` is exactly `target` bytes (protobuf runtime)."""
    from tests import _wire as W

    lo, hi = 0, 1 << 17
    while lo < hi:
        mid = (lo + hi) // 2
        if W.message_pack(ch, b"\0" * mid).ByteSize() < target:
            lo = mid + 1
        else:
            hi = mid
    assert W.message_pack(ch, b"\0" * lo).ByteSize() == target
    return lo


class Payload:
    """The engine's payload stage with host buffers that grow on demand: chd_set_payload_bytes, chd_assemble_payloads,
    chd_frame_packets, chd_due_classes."""

    def __init__(self, chd, e, n_slots):
        self.capi, self.e, self.S = chd.capi, e, n_slots
        self.cls_off = np.zeros(int(e.lim.max_due) + 2, np.uint64)  # calloc'd: only the used part is touched
        self.blob = np.zeros(1 << 20, np.uint8)
        self.out = np.zeros(1 << 24, np.uint8)
        self.conn_off = np.zeros(n_slots + 1, np.uint64)
        self.conn_len = np.zeros(n_slots, np.uint32)
        self.conn_frames = np.zeros(n_slots, np.uint32)

    def set_bytes(self, entry_off, entry_bytes, full_off, full_bytes):
        from tests import _wire as W

        capi, e = self.capi, self.e
        self._keep = [np.ascontiguousarray(a) for a in (entry_off, entry_bytes, full_off, full_bytes)]
        eo, eb, fo, fb = (a if len(a) else np.zeros(1, a.dtype) for a in self._keep)
        st = e.L.chd_set_payload_bytes(e.h, capi.ptr(eo), len(entry_off) - 1, capi.ptr(eb), capi.ptr(fo), capi.ptr(fb), W.TYPE_URL.encode(),
                                       W.MSG_CHANNEL_DATA_UPDATE)
        assert st == capi.OK, e.L.chd_last_error(e.h)

    def assemble(self):
        """-> (n_classes, class_off[n_classes + 1], blob)"""
        capi, e = self.capi, self.e
        while True:
            ncls, blen = C.c_uint32(), C.c_uint64()
            st = e.L.chd_assemble_payloads(e.h, C.byref(ncls), capi.ptr(self.cls_off), len(self.cls_off) - 1, capi.ptr(self.blob), self.blob.size,
                                           C.byref(blen))
            if st == capi.ERR_CAPACITY and blen.value > self.blob.size:
                self.blob = np.zeros(blen.value + blen.value // 4, np.uint8)
                continue
            assert st == capi.OK, e.L.chd_last_error(e.h)
            k = ncls.value
            return k, self.cls_off[:k + 1].copy() if k else np.zeros(1, np.uint64), self.blob[:blen.value]

    def frame(self, compression):
        """-> (conn_off, conn_len, conn_frames, out bytes, n_dropped)"""
        capi, e = self.capi, self.e
        comp = np.ascontiguousarray(compression, np.uint8)
        while True:
            olen, dropped = C.c_uint64(), C.c_uint32()
            st = e.L.chd_frame_packets(e.h, capi.ptr(comp), capi.ptr(self.conn_off), capi.ptr(self.conn_len), capi.ptr(self.conn_frames),
                                       capi.ptr(self.out), self.out.size, C.byref(olen), C.byref(dropped))
            if st == capi.ERR_CAPACITY and olen.value > self.out.size:
                self.out = np.zeros(olen.value + olen.value // 4, np.uint8)
                continue
            assert st == capi.OK, e.L.chd_last_error(e.h)
            assert olen.value == int(self.conn_off[self.S])
            return self.conn_off.copy(), self.conn_len.copy(), self.conn_frames.copy(), self.out[:olen.value], dropped.value


def check_classes(cls_of, cls_rep, cls_cnt, real):
    """class_of covers exactly [0, n_classes) over the real decisions (holes: CHD_DUE_VOID), class_rep[k] is the lowest member
    of class k, class_count[k] its size, and the reps ascend."""
    from channeld_b200 import capi

    K = len(cls_rep)
    assert len(cls_cnt) == K
    assert (cls_of[~real] == capi.DUE_VOID).all(), "a hole was classified"
    co = cls_of[real].astype(np.int64)
    assert co.size == 0 or co.max() < K, "a class id outside [0, n_classes)"
    cnt = np.bincount(co, minlength=K)
    assert (cnt > 0).all(), "an empty class"
    np.testing.assert_array_equal(cls_cnt, cnt)
    ids, first = np.unique(co, return_index=True)
    np.testing.assert_array_equal(cls_rep, np.nonzero(real)[0][first])
    assert (np.diff(cls_rep.astype(np.int64)) > 0).all()


def restate_frames(sub, due_idx, cls_of, cls_len, n_slots, compression):
    """connection.go's Send / flush restated on entry lengths (a Packet's size is the sum of its entries, a MessagePack at the
    drop limit is dropped, a message that would overflow the packet opens the next one), per connection over its decisions in
    ascending due index.  -> dict(kept: due indices in (connection, due index) order, pk_conn, pk_begin / pk_end (ranges of
    kept), pk_len, pk_comp, n_dropped)"""
    order = np.lexsort((due_idx, sub))
    L = cls_len[cls_of[order]].astype(np.int64)
    drop = L >= DROP_ENTRY
    kept, Lk = order[~drop], L[~drop]
    sk = sub[kept].astype(np.int64)
    tot = np.bincount(sk, weights=Lk, minlength=n_slots).astype(np.int64)
    cb = np.searchsorted(sk, np.arange(n_slots + 1))
    one = np.nonzero((tot > 0) & (tot <= PKT_MAX))[0]
    pk = [(one, cb[one], cb[one + 1], tot[one])]
    for s in np.nonzero(tot > PKT_MAX)[0]:  # several packets: the greedy cut, literally
        b, cur, rows = cb[s], 0, []
        for a in range(cb[s], cb[s + 1]):
            if cur + Lk[a] > PKT_MAX:
                rows.append((s, b, a, cur))
                b, cur = a, 0
            cur += Lk[a]
        rows.append((s, b, cb[s + 1], cur))
        pk.append(tuple(np.array(c, np.int64) for c in zip(*rows)))
    pk_conn, pk_begin, pk_end, pk_len = (np.concatenate([p[i] for p in pk]).astype(np.int64) for i in range(4))
    o = np.lexsort((pk_begin, pk_conn))
    comp = np.asarray(compression)[pk_conn[o]] == 1
    return dict(kept=kept, kept_cls=cls_of[kept], kept_len=Lk, pk_conn=pk_conn[o], pk_begin=pk_begin[o], pk_end=pk_end[o], pk_len=pk_len[o], pk_comp=comp,
                n_dropped=int(drop.sum()))


def check_frames(r, cls_off, blob, frames, n_slots, compression):
    """Every connection's bytes against the restated flush: tags, size fields, raw bodies byte for byte, snappy bodies through
    pyarrow's decoder, the raw fallback only where the encoding may not fit, conn_frames, n_dropped and the reservation."""
    conn_off, conn_len, conn_frames, out, dropped = frames
    assert dropped == r["n_dropped"]
    pk_conn, pk_len, pk_comp = r["pk_conn"], r["pk_len"], r["pk_comp"]
    np.testing.assert_array_equal(conn_frames, np.bincount(pk_conn, minlength=n_slots))
    res = 5 + np.where(pk_comp, 32 + pk_len + pk_len // 6, pk_len)
    np.testing.assert_array_equal(np.diff(conn_off.astype(np.int64)), np.bincount(pk_conn, weights=res, minlength=n_slots).astype(np.int64))
    assert (conn_len <= np.diff(conn_off.astype(np.int64))).all()
    # the expected bodies: the kept entries in (connection, due index) order, packet after packet
    stream = _gather(blob, cls_off[r["kept_cls"]].astype(np.int64), r["kept_len"])
    pk_off = np.concatenate([[0], np.cumsum(pk_len)])
    assert pk_off[-1] == len(stream)
    # raw connections: tag + body per packet, every byte
    raw = np.asarray(compression)[np.arange(n_slots)] != 1
    pr = np.nonzero(~pk_comp)[0]
    tags = np.zeros((len(pr), 5), np.uint8)
    tags[:, 0], tags[:, 1], tags[:, 2], tags[:, 3] = 67, 72, pk_len[pr] >> 8, pk_len[pr] & 0xFF
    src = np.concatenate([stream, tags.reshape(-1)])
    seg_start = np.stack([len(stream) + 5 * np.arange(len(pr)), pk_off[pr]], 1).reshape(-1)
    seg_len = np.stack([np.full(len(pr), 5), pk_len[pr]], 1).reshape(-1)
    want_raw = _gather(src, seg_start, seg_len)
    want_len = np.bincount(pk_conn[pr], weights=5 + pk_len[pr], minlength=n_slots).astype(np.int64)
    np.testing.assert_array_equal(conn_len[raw], want_len[raw])
    rs = np.nonzero(raw)[0]
    got_raw = _gather(out, conn_off[rs].astype(np.int64), conn_len[rs])
    if not np.array_equal(got_raw, want_raw):
        bad = rs[np.searchsorted(np.cumsum(conn_len[rs].astype(np.int64)), np.argmax(got_raw != want_raw), side="right")]
        raise AssertionError("raw frames of connection slot %d differ from the restated flush" % bad)
    # snappy connections: parse like connection.go's reader; every body decodes to its packet
    ob, sb = out.tobytes(), stream.tobytes()
    first = np.searchsorted(pk_conn, np.arange(n_slots + 1))
    n_snappy = n_raw_fallback = 0
    for s in np.nonzero(~raw)[0].tolist():
        pos, end = int(conn_off[s]), int(conn_off[s]) + int(conn_len[s])
        for p in range(first[s], first[s + 1]):
            assert ob[pos:pos + 2] == b"CH", s
            size, ct = (ob[pos + 2] << 8) | ob[pos + 3], ob[pos + 4]
            body, want = ob[pos + 5:pos + 5 + size], sb[pk_off[p]:pk_off[p + 1]]
            assert len(body) == size > 0, s
            if ct == 1:
                assert _snappy_decode(body) == want, s
                n_snappy += 1
            else:
                assert ct == 0 and body == want and len(want) > SNAPPY_FITS_UP_TO, s
                n_raw_fallback += 1
            pos += 5 + size
        assert pos == end, s
    return n_snappy, n_raw_fallback


def _run_case(chd, oracle, case):
    from tests import _wire as W
    from tests._oracle import make_grid

    capi = chd.capi
    grid = case[0]
    g = GRIDS[grid]
    offx, offz, w, h, cols, rows = g
    Cn = cols * rows
    Wd, Hd = w * cols, h * rows
    og = make_grid(*g)
    rng = np.random.default_rng({"a": 41, "e": 42, "a-tick": 43}[case])
    S = 100_000
    conn = np.arange(1, S + 1, dtype=np.uint32)
    cx, cz = offx + rng.random(S) * Wd, offz + rng.random(S) * Hd
    rad = rng.choice(RADII[grid], S)
    heavy = np.arange(HEAVY) * (S // HEAVY) + 7
    cx[heavy] = offx + Wd * rng.uniform(0.4, 0.6, HEAVY)
    cz[heavy] = offz + Hd * rng.uniform(0.4, 0.6, HEAVY)
    rad[heavy] = HEAVY_R[grid]
    moves = np.ones(S, bool)
    moves[heavy] = False
    compression = (np.arange(S) % 2).astype(np.uint8)  # every other connection asked for snappy
    ex, ez = np.array([offx + 1.0]), np.array([offz + 1.0])
    e = chd.engine.Engine(chd.engine.grid_cfg(*g), 1, S, max_pairs=2 << 20, max_due=8 << 20, max_ring_entries=Cn * 64 + (1 << 17),
                          max_window_cells=S * 32 + 65536)
    e.enable_graphs(True)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    e.build()
    pl = Payload(chd, e, S)
    chans = oracle.channels(Cn)
    # opaque payload bytes: slices of a pool, half random (snappy literals), half repetitive text (snappy copies)
    pool = np.concatenate([np.frombuffer(rng.bytes(1 << 20), np.uint8), np.frombuffer((b"position update for entity 12345; " * 31000)[:1 << 20], np.uint8)])

    def slices(n, max_len):
        return rng.integers(0, len(pool) - max_len, n), (rng.random(n) ** 3 * (max_len + 1)).astype(np.int64)

    f_src, f_len = slices(Cn, 200)
    special = rng.choice(Cn, 6, replace=False)
    big, drop = special[:4], special[4:]
    big_len = rng.integers(20000, 40001, len(big))
    f_src[big] = rng.integers(0, len(pool) - 40001, len(big))
    drop_len = [_value_len_for_mp(MP_DROP, S0 + int(drop[0])), _value_len_for_mp(MP_DROP + 700, S0 + int(drop[1]))]
    f_src[drop] = rng.integers(0, len(pool) - 70000, 2)
    f_len[drop] = drop_len
    big_from = 2 if grid == "a" else 0  # the benchmark grid's cells have thousands of subscribers: big data on new pairs only
    r_cell = np.zeros(0, np.uint32); r_arr = np.zeros(0, np.int64); r_snd = np.zeros(0, np.uint32); r_idx = np.zeros(0, np.uint64)
    r_src = np.zeros(0, np.int64); r_len = np.zeros(0, np.int64)
    msg_index = np.zeros(Cn, np.uint64)
    bench_state = None
    prev_keys = np.zeros(0, np.int64)
    t = 0
    st = dict(max_due=0, max_cls=0, remade=False, heavy_split=0, dropped=0, snappy=0, raw_fallback=0, update_cls=0, multi_tile=False)
    cls_before = 0
    t_case = time.time()
    for tick in range(N_TICKS):
        gap = 70 * MS if tick % 3 == 0 else 33 * MS  # irregular ticks: 20 ms pairs fall several intervals behind
        t += gap
        if tick:
            mv = moves & (rng.random(S) < 0.3)
            cx[mv] = np.clip(cx[mv] + rng.uniform(-0.6, 0.6, mv.sum()) * w, offx + 1e-3, offx + Wd - 1e-3)
            cz[mv] = np.clip(cz[mv] + rng.uniform(-0.6, 0.6, mv.sum()) * h, offz + 1e-3, offz + Hd - 1e-3)
        # ---- interest (the oracle channels follow the wanted pairs)
        want = oracle.sphere_pairs(og, ex, ez, cx, cz, rad)
        assert (want["status"] == 0).all()
        P = len(want["pair_cell"])
        w_sub = np.repeat(np.arange(S), np.diff(want["pair_off"].astype(np.int64)))
        w_cell = want["pair_cell"].astype(np.int64) - S0
        w_iv = np.select([want["pair_dist"] == 0, want["pair_dist"] == 1, want["pair_dist"] == 2], [20, 50, 100], 20).astype(np.uint32)
        keys = (w_sub.astype(np.int64) << 20) | w_cell
        gone = np.setdiff1d(prev_keys, keys)
        chans.unsubscribe(gone & 0xFFFFF, conn[gone >> 20])
        chans.subscribe(w_cell, conn[w_sub], t, w_iv)
        prev_keys = np.sort(keys)
        if tick == 0:
            assert np.diff(want["pair_off"].astype(np.int64))[heavy].min() >= 200
        # ---- update rings (as tests/test_gpu_fanout_scale.py builds them) and their payload bytes
        if grid == "a":
            bench_state, _, _, _, _, _ = chd.synth.update_rings(chd.synth.CONFIGS["benchmark"], tick, t, gap, 8, S, ring_len=512, state=bench_state)
            n_cell = np.full(Cn, 8)
        else:
            n_cell = rng.integers(0, 9, Cn)
        n_new = int(n_cell.sum())
        u_cell = np.repeat(np.arange(Cn, dtype=np.uint32), n_cell)
        if grid == "a":
            u_arr = bench_state["arrival"][:, -8:].reshape(-1)
            u_snd = bench_state["sender"][:, -8:].reshape(-1)
        else:
            u_arr = t - rng.integers(0, 80, n_new) * MS
            bc = np.sort(w_cell, kind="stable")
            bs = w_sub[np.argsort(w_cell, kind="stable")]
            cs = np.searchsorted(bc, np.arange(Cn + 1))
            cnt = np.diff(cs)[u_cell]
            pick = cs[u_cell] + (rng.random(n_new) * np.maximum(cnt, 1)).astype(np.int64)
            u_snd = np.where((rng.random(n_new) < 0.5) & (cnt > 0), conn[bs[np.minimum(pick, len(bs) - 1)]], 7).astype(np.uint32)
        u_arr, u_snd = np.asarray(u_arr, np.int64), np.asarray(u_snd, np.uint32)
        first_idx = np.concatenate([[0], np.cumsum(n_cell)[:-1]])
        u_idx = msg_index[u_cell] + 1 + (np.arange(n_new) - first_idx[u_cell]).astype(np.uint64)
        msg_index += n_cell.astype(np.uint64)
        chans.on_update(u_cell, u_arr, u_snd)
        u_src, u_len = slices(n_new, 300)
        r_cell = np.concatenate([r_cell, u_cell]); r_arr = np.concatenate([r_arr, u_arr]); r_snd = np.concatenate([r_snd, u_snd])
        r_idx = np.concatenate([r_idx, u_idx]); r_src = np.concatenate([r_src, u_src]); r_len = np.concatenate([r_len, u_len])
        o = np.argsort(r_cell, kind="stable")
        r_cell, r_arr, r_snd, r_idx, r_src, r_len = r_cell[o], r_arr[o], r_snd[o], r_idx[o], r_src[o], r_len[o]
        ring_off = np.searchsorted(r_cell, np.arange(Cn + 1)).astype(np.int64)
        assert np.diff(ring_off).max() <= 512  # the oracle's eviction never fires
        e.set_rings(ring_off.astype(np.uint32), r_arr, r_snd, r_idx, msg_index)
        fl = f_len.copy()
        if tick >= big_from:
            fl[big] = big_len
        eoff = np.concatenate([[0], np.cumsum(r_len)]).astype(np.uint64)
        foff = np.concatenate([[0], np.cumsum(fl)]).astype(np.uint64)
        eb, fb = _gather(pool, r_src, r_len), _gather(pool, f_src, fl)
        pl.set_bytes(eoff, eb, foff, fb)
        # ---- the tick, then the byte half
        batch, keep = chd.engine.make_batch(S, sphere=(cx, cz, rad))
        if case == "a-tick":
            e.tick(batch, t, capi.TICK_ALL, want_summary=False)  # the visible-list copy runs on its own stream
        else:
            e.update_interest(batch, t)
            e.fanout_tick(t)
        n_cls, cls_off, blob = pl.assemble()
        frames = pl.frame(compression)
        s = e.summary()
        assert s.overflow == 0 and s.n_pairs == P
        n_due = int(s.n_due)
        cls_of, cls_rep, cls_cnt = e.due_classes(n_due)
        assert len(cls_rep) == n_cls
        due = e.get_due(n_due)
        # ---- the oracle's decisions with their identities; device record i <-> oracle send j
        sends, soff, lo, sk, sel_off, sel_pos = chans.tick_data_ex(t, 4 * P + 4096, 1 << 27)
        assert len(sends) == n_due
        s_chan = np.repeat(np.arange(Cn, dtype=np.int64), np.diff(soff.astype(np.int64)))
        d_chan = due["channel_id"].astype(np.int64) - S0
        d_conn = conn[due["sub"]].astype(np.int64)
        oo = np.lexsort((sends["window_hi"], s_chan, sends["conn_id"]))
        do = np.lexsort((due["window_hi"], d_chan, d_conn))
        for a, b in [(d_conn, sends["conn_id"]), (d_chan, s_chan), (due["kind"], sends["kind"]), (due["window_hi"], sends["window_hi"]),
                     (due["n_selected"], sends["n_selected"]), (due["first_sel"], sends["first_sel"]), (due["last_sel"], sends["last_sel"]),
                     (due["sel_hash"], sends["sel_hash"]), (due["last_message_index"], sends["last_message_index"])]:
            np.testing.assert_array_equal(np.asarray(a)[do].astype(np.int64), np.asarray(b)[oo].astype(np.int64))
        j_of = np.empty(n_due, np.int64)
        j_of[do] = oo
        # ---- classes
        real = np.ones(n_due, bool)
        check_classes(cls_of, cls_rep, cls_cnt, real)
        full = due["kind"] == 0
        nsel = np.diff(sel_off.astype(np.int64))[j_of]
        ident = np.stack([d_chan, full, np.where(full, 0, lo[j_of]), np.where(full, 0, due["window_hi"]),
                          np.where(full | (sk[j_of] == 0), 0, d_conn)], 1)
        io = np.lexsort(ident.T[::-1])
        new_ident = np.concatenate([np.ones(min(n_due, 1), bool), (np.diff(ident[io], axis=0) != 0).any(1)])
        assert int(new_ident.sum()) == n_cls, "classes are not the payload identities"
        same_ident = ~new_ident[1:]
        assert (cls_of[io][1:][same_ident] == cls_of[io][:-1][same_ident]).all(), "an identity is split over two classes"
        rep_of = cls_rep[cls_of].astype(np.int64)  # no class mixes two exact payloads: every member's equals its rep's
        assert (d_chan == d_chan[rep_of]).all() and (full == full[rep_of]).all() and (nsel == nsel[rep_of]).all()
        upd = np.nonzero(~full)[0]
        np.testing.assert_array_equal(_gather(sel_pos, sel_off[j_of[upd]], nsel[upd]), _gather(sel_pos, sel_off[j_of[rep_of[upd]]], nsel[upd]))
        # ---- class entries: once per class, from the oracle's selection of its rep
        kr = cls_rep.astype(np.int64)
        c_k, full_k, n_k = d_chan[kr], full[kr], nsel[kr]
        nseg = np.where(full_k, 1, n_k)
        seg_cls = np.repeat(np.arange(n_cls), nseg)
        within = np.arange(len(seg_cls)) - np.repeat(np.cumsum(nseg) - nseg, nseg)
        is_full = full_k[seg_cls]
        pos = sel_pos[sel_off[j_of[kr[seg_cls[~is_full]]]].astype(np.int64) + within[~is_full]]
        gidx = ring_off[c_k[seg_cls[~is_full]]] + pos
        seg_start, seg_len = np.zeros(len(seg_cls), np.int64), np.zeros(len(seg_cls), np.int64)
        seg_start[~is_full], seg_len[~is_full] = eoff[gidx].astype(np.int64), r_len[gidx]
        cf = c_k[seg_cls[is_full]]
        seg_start[is_full], seg_len[is_full] = len(eb) + foff[cf].astype(np.int64), fl[cf]
        vals = _gather(np.concatenate([eb, fb]), seg_start, seg_len).tobytes()
        voff = np.concatenate([[0], np.cumsum(np.bincount(seg_cls, weights=seg_len, minlength=n_cls).astype(np.int64))])
        want_entries = [W.class_entry(int(c_k[k]) + S0, vals[voff[k]:voff[k + 1]]) for k in range(n_cls)]
        np.testing.assert_array_equal(np.diff(cls_off.astype(np.int64)), [len(x) for x in want_entries])
        assert int(cls_off[-1]) == len(blob)
        if blob.tobytes() != b"".join(want_entries):
            bad = next(k for k in range(n_cls) if blob[int(cls_off[k]):int(cls_off[k + 1])].tobytes() != want_entries[k])
            raise AssertionError("class %d (channel %d, kind %d) entry differs" % (bad, c_k[bad] + S0, not full_k[bad]))
        # ---- frames
        cls_len = np.diff(cls_off.astype(np.int64))
        r = restate_frames(due["sub"], np.arange(n_due), cls_of.astype(np.int64), cls_len, S, compression)
        n_snappy, n_fallback = check_frames(r, cls_off, blob, frames, S, compression)
        # ---- what this tick exercised
        dec = np.bincount(due["sub"], minlength=S)
        st["heavy_split"] = max(st["heavy_split"], int((dec[frames[2] > 1]).max(initial=0)))
        st["max_due"], st["dropped"] = max(st["max_due"], n_due), st["dropped"] + frames[4]
        st["multi_tile"] |= n_due > SCAN_TILE and n_cls > SCAN_TILE
        st["remade"] |= cls_before > 0 and n_cls > 1.25 * cls_before + SCAN_TILE
        cls_before = max(cls_before, n_cls)
        st["max_cls"] = max(st["max_cls"], n_cls)
        st["update_cls"] = max(st["update_cls"], int((~full_k).sum()))
        st["snappy"] += n_snappy
        st["raw_fallback"] += n_fallback
    e.close()
    print("payload scale %s: %.1f s, %s" % (case, time.time() - t_case, st))
    return st


@pytest.mark.parametrize("case", ["a", "e", "a-tick"])
def test_payload_scale_parity(chd, oracle, case):
    st = _run_case(chd, oracle, case)
    # the paths each case is built to take.  S = 100 000 > SCAN_TILE: both frame scans span several tiles in every case, and
    # the class numbering scan runs over the due list
    assert st["max_due"] > SCAN_TILE, st
    assert st["heavy_split"] >= 200, st  # a connection with at least 200 decisions in more than one packet
    assert st["dropped"] > 0 and st["snappy"] > 0, st
    if case[0] == "a":
        assert st["update_cls"] > 2000, st  # many UPDATE classes
    else:
        assert st["multi_tile"], st  # more than 4 096 classes: the class-length scan spans several tiles
        assert st["remade"], st      # a class count outgrew the class-length scan's site: remake_site rebuilt it


def test_overflowed_due_list_holes_are_in_no_class(chd, oracle):
    """A due list that overflows holds CHD_DUE_VOID holes with whatever key an earlier tick left in their slots.  Holes belong to
    no class; the classes, the class entries and every connection's frames cover the real decisions only.

    A pair whose decisions do not all fit leaves holes, so holes need pairs with two decisions: a first fan-out (FULL) is always
    a pair's only decision in its tick.  Tick A: M = 1001 SpotsAOI pairs (20 ms interval) get their FULL, which fills the due
    list (max_due = M) exactly: every key slot now holds a valid FULL key.  Tick B, 40 ms later: every pair is two intervals
    behind, and each window holds one ring entry of its channel (arrivals 10 ms and 30 ms into the gap), so every pair makes two
    UPDATE decisions.  Block reservations are even and M is odd, so the list is M - 1 decisions and one hole, at M - 1.  The
    pairs that did not fit are untouched and catch up in the next ticks, each window delivered once."""
    from tests import _wire as W

    capi = chd.capi
    n_cells, n_conn, per = 64, 143, 7
    M = n_conn * per
    assert M % 2 == 1
    subs = [sorted({(5 * j + 9 * k) % n_cells for k in range(per)}) for j in range(n_conn)]
    assert all(len(c) == per for c in subs)
    conn = np.arange(101, 101 + n_conn, dtype=np.uint32)
    e = chd.engine.Engine(chd.engine.grid_cfg(0, 0, 10, 10, n_cells, 1), 8, n_conn, max_due=M)
    e.set_subscribers(conn)
    e.set_entities(np.array([5.0]), np.array([5.0]))
    e.build()
    n_sp = np.full(n_conn, per, np.uint32)
    off = np.concatenate([[0], np.cumsum(n_sp)]).astype(np.uint32)
    x = np.array([10.0 * c + 5.0 for cs in subs for c in cs])
    batch, keep = chd.engine.make_batch(n_conn, sub=np.arange(n_conn, dtype=np.uint32), kind=np.full(n_conn, capi.AOI_SPOTS, np.uint8),
                                        spots=(off, n_sp, x, np.full(len(x), 5.0), np.zeros(len(x), np.uint32)))
    e.update_interest(batch, 0)
    assert e.summary().n_pairs == M
    pl = Payload(chd, e, n_conn)
    rng = np.random.default_rng(77)
    fulls = [rng.bytes(int(rng.integers(0, 200))) if c % 2 else (b"full data of channel %d; " % c) * int(rng.integers(1, 12))
             for c in range(n_cells)]
    foff = np.concatenate([[0], np.cumsum([len(b) for b in fulls])]).astype(np.uint64)
    fb = np.frombuffer(b"".join(fulls), np.uint8)
    compression = (np.arange(n_conn) % 2).astype(np.uint8)
    tA, tB = 100 * MS, 140 * MS
    entries = {}  # (cell, window_hi) -> the bytes of the one ring entry in that window

    def run(t, ring):
        """ring: per cell [(arrival, bytes)] -> (due, real mask, n_due as reported, overflow)"""
        roff = np.concatenate([[0], np.cumsum([len(r) for r in ring])]).astype(np.uint32)
        flat = [x for r in ring for x in r]
        e.set_rings(roff, np.array([a for a, _ in flat], np.int64), np.full(len(flat), 7, np.uint32),
                    np.array([k + 1 for r in ring for k in range(len(r))], np.uint64), np.array([len(r) for r in ring], np.uint64))
        eoff = np.concatenate([[0], np.cumsum([len(b) for _, b in flat])]).astype(np.uint64)
        pl.set_bytes(eoff, np.frombuffer(b"".join(b for _, b in flat), np.uint8), foff, fb)
        e.fanout_tick(t)
        s = capi.TickSummary()
        assert e.L.chd_summary(e.h, C.byref(s)) == (capi.ERR_CAPACITY if s.overflow else capi.OK)
        n_list = min(int(s.n_due), M)
        due = e.get_due(n_list)
        real = due["kind"] != capi.DUE_VOID
        n_cls, cls_off, blob = pl.assemble()
        cls_of, cls_rep, cls_cnt = e.due_classes(n_list)
        frames = pl.frame(compression)
        # the classes partition the real decisions: one per (channel, kind, window) among them
        check_classes(cls_of, cls_rep, cls_cnt, real)
        ident = {(int(d["channel_id"]), int(d["kind"]), int(d["window_hi"]) if d["kind"] else 0) for d in due[real]}
        assert n_cls == len(ident)
        # every real decision's entry
        for i in np.nonzero(real)[0]:
            d = due[i]
            c = int(d["channel_id"]) - S0
            value = fulls[c] if d["kind"] == 0 else entries[(c, int(d["window_hi"]))]
            k = int(cls_of[i])
            assert blob[int(cls_off[k]):int(cls_off[k + 1])].tobytes() == W.class_entry(S0 + c, value), i
        assert int(cls_off[-1]) == len(blob)
        # every connection's frames: the literal flush of its real decisions' entries, in ascending due index
        conn_off, conn_len, conn_frames, out, dropped = frames
        n_drop = 0
        for j in range(n_conn):
            mine = [i for i in np.nonzero(real & (due["sub"] == j))[0]]
            packets, dr = W.flush([W.Packet.FromString(blob[int(cls_off[cls_of[i]]):int(cls_off[cls_of[i] + 1])].tobytes()).messages[0]
                                   for i in mine])
            n_drop += dr
            buf = out[int(conn_off[j]):int(conn_off[j]) + int(conn_len[j])].tobytes()
            pos = 0
            for p in packets:
                assert buf[pos:pos + 2] == b"CH"
                size, ct = (buf[pos + 2] << 8) | buf[pos + 3], buf[pos + 4]
                body = buf[pos + 5:pos + 5 + size]
                assert (_snappy_decode(body) if ct == 1 else body) == p and ct == compression[j], j
                pos += 5 + size
            assert pos == len(buf) and conn_frames[j] == len(packets), j
        assert dropped == n_drop == 0
        return due, real, int(s.n_due), s.overflow, cls_of

    # tick A: every pair's FULL, exactly max_due decisions
    due, real, n_due, ovf, _ = run(tA, [[] for _ in range(n_cells)])
    assert n_due == M and ovf == 0 and real.all() and (due["kind"] == 0).all()
    # ticks B, C, ...: two UPDATE windows per pair, one ring entry in each
    ring = []
    for c in range(n_cells):
        a, b = rng.bytes(int(rng.integers(1, 300))), rng.bytes(int(rng.integers(1, 300)))
        entries[(c, tA + 20 * MS)], entries[(c, tA + 40 * MS)] = a, b
        ring.append([(tA + 10 * MS, a), (tA + 30 * MS, b)])
    delivered, needed, t = [], [], tB
    for step in range(4):
        due, real, n_due, ovf, cls_of = run(t, ring)
        holes = np.nonzero(~real)[0]
        assert (cls_of[holes] == capi.DUE_VOID).all()
        if ovf:
            assert ovf == capi.OVF_DUE and holes.tolist() == [M - 1], (n_due, holes[:8])
        else:
            assert len(holes) == 0
        needed.append(n_due)
        assert (due["kind"][real] == 1).all()
        delivered += list(zip(due["sub"][real].tolist(), due["channel_id"][real].tolist(), due["window_hi"][real].tolist()))
        if not ovf:
            break
        t += 5 * MS
    # B: 2 M decisions, M - 1 fit; C: the other (M + 1) / 2 pairs, all but one fit; D: the last pair
    assert needed == [2 * M, M + 1, 2]
    want = sorted((j, S0 + c, tA + k * 20 * MS) for j in range(n_conn) for c in subs[j] for k in (1, 2))
    assert sorted(delivered) == want  # every window delivered once: nothing lost, nothing twice
    e.close()
