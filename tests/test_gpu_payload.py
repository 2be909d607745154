"""GPU test of the byte half of the fan-out (chd_set_payload_bytes / chd_assemble_payloads / chd_frame_packets, SURVEY.md §8f
rank 1 and 4).  The merge is checked at MESSAGE level (Go's merged value has no defined byte form, SURVEY §8c): the bytes the
device assembles are decoded with the protobuf runtime and compared with proto.Merge (MergeFrom) over the ring entries the
literal tickData emulation (oracle channel) actually merged.  The wrapper layers are fixed proto3 encodings, so class entries
are also compared byte for byte with the protobuf runtime's serialization, and the framed packets byte for byte with a
restatement of connection.go's Send / flush (tests/_wire.py) at the 64 KB edges; frames are parsed like connection.go's
reader does (5-byte tag, snappy via an independent decoder: pyarrow's)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
S0 = 65536
MS = 1_000_000


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


def test_payload_assembly_and_framing(chd, oracle):
    from tests import _wire as W
    from tests._oracle import make_grid

    capi = chd.capi
    g = (-300.0, -250.0, 100.0, 100.0, 6, 5)
    og = make_grid(*g)
    rng = np.random.default_rng(5)
    S, N = 40, 200
    cells = g[4] * g[5]
    e = chd.engine.Engine(chd.engine.grid_cfg(*g), N, S, max_visible=1 << 20)
    conn = np.arange(101, 101 + S, dtype=np.uint32)
    e.set_subscribers(conn)
    e.set_entities(rng.uniform(-300, 300, N), rng.uniform(-250, 250, N))
    e.build()
    chans = [oracle.channel() for _ in range(cells)]
    rings = [[] for _ in range(cells)]      # (arrival, sender, index, message)
    full = [W.TestChannelDataMessage() for _ in range(cells)]  # ch.data.msg: every update merged in (data.go:149-160)
    msg_index = np.zeros(cells, np.uint64)
    cx, cz = rng.uniform(-280, 280, S), rng.uniform(-230, 230, S)
    rad = rng.choice([30.0, 60.0, 120.0], S)
    compression = (np.arange(S) % 2).astype(np.uint8)  # every other connection asked for snappy
    t = 0
    n_checked = n_update_msgs = n_shared = n_multi_frame = 0
    for tick in range(10):
        t += 33 * MS if tick % 3 else 90 * MS
        cx += rng.uniform(-40, 40, S)
        cz += rng.uniform(-40, 40, S)
        batch, keep = chd.engine.make_batch(S, sphere=(cx, cz, rad))
        e.update_interest(batch, t)
        s = e.summary()
        pairs = e.get_pairs()
        for j in range(S):
            res, st = oracle.query(og, sphere=(cx[j], cz[j], rad[j]))
            if st != 0:
                continue
            have = set(int(c) for c in pairs["channel"][pairs["off"][j]:pairs["off"][j + 1]])
            for c in range(cells):
                ch = S0 + c
                if ch in res:
                    chans[c].subscribe(int(conn[j]), t, oracle.damping(res[ch], 20), 0, True, False)
                else:
                    chans[c].unsubscribe(int(conn[j]))
            assert have == set(res.keys())
        for _ in range(int(rng.integers(10, 40))):
            c = int(rng.integers(0, cells))
            arrival = t - int(rng.integers(0, 60)) * MS
            sender = int(rng.choice(conn)) if rng.random() < 0.4 else 7
            m = W.TestChannelDataMessage()
            if rng.random() < 0.7:
                m.text = "t%d-%d" % (tick, int(rng.integers(0, 1000)))
            if rng.random() < 0.5:
                m.num = int(rng.integers(1, 1 << 20))
            for _k in range(int(rng.integers(0, 3))):
                m.list.append("e%d" % int(rng.integers(0, 100)))
            for _k in range(int(rng.integers(0, 3))):
                m.kv[int(rng.integers(0, 6))] = "v%d" % int(rng.integers(0, 100))
            msg_index[c] += 1
            rings[c].append((arrival, sender, int(msg_index[c]), m))
            full[c].MergeFrom(m)
            chans[c].on_update(arrival, sender)
        ring_off = np.concatenate([[0], np.cumsum([len(r) for r in rings])]).astype(np.uint32)
        flat = [x for r in rings for x in r]
        e.set_rings(ring_off, np.array([f[0] for f in flat], np.int64), np.array([f[1] for f in flat], np.uint32),
                    np.array([f[2] for f in flat], np.uint64), msg_index)
        ebytes = [f[3].SerializeToString() for f in flat]
        eoff = np.concatenate([[0], np.cumsum([len(b) for b in ebytes])]).astype(np.uint64)
        fbytes = [m.SerializeToString() for m in full]
        foff = np.concatenate([[0], np.cumsum([len(b) for b in fbytes])]).astype(np.uint64)
        eb = np.frombuffer(b"".join(ebytes) or b"\0", np.uint8).copy()
        fb = np.frombuffer(b"".join(fbytes) or b"\0", np.uint8).copy()
        st_ = e.L.chd_set_payload_bytes(e.h, capi.ptr(eoff), len(flat), capi.ptr(eb), capi.ptr(foff), capi.ptr(fb), W.TYPE_URL.encode(),
                                         W.MSG_CHANNEL_DATA_UPDATE)
        assert st_ == capi.OK, e.L.chd_last_error(e.h)
        e.fanout_tick(t)
        s = e.summary()
        due = e.get_due(s.n_due)
        # ---- what the reference would send: per (conn, channel, step) the merge of the entries the emulation picked
        want = {}
        for c in range(cells):
            for d in chans[c].tick_data_ex(t):
                if d["kind"] == 0:
                    m = W.TestChannelDataMessage()
                    m.CopyFrom(full[c])
                else:
                    m = W.TestChannelDataMessage()
                    for pos in d["selected"]:
                        m.MergeFrom(rings[c][pos][3])  # proto.Merge of every selected entry, in order (data.go:246-256)
                    n_update_msgs += 1
                want.setdefault((d["conn"], S0 + c), []).append(m)
        # ---- per-class blobs
        ncls = C.c_uint32()
        blob_len = C.c_uint64()
        cap_cls = max(int(s.n_due), 1)
        cls_off = np.zeros(cap_cls + 1, np.uint64)
        blob = np.zeros(1 << 22, np.uint8)
        st_ = e.L.chd_assemble_payloads(e.h, C.byref(ncls), capi.ptr(cls_off), cap_cls, capi.ptr(blob), blob.size, C.byref(blob_len))
        assert st_ == capi.OK, e.L.chd_last_error(e.h)
        cls_of, cls_rep, cls_cnt = e.due_classes(int(s.n_due))
        assert len(cls_rep) == ncls.value
        n_shared += int(s.n_due) - ncls.value
        got = {}
        for i, d in enumerate(due):
            k = int(cls_of[i])
            entry = bytes(blob[int(cls_off[k]):int(cls_off[k + 1])])
            pk = W.Packet()
            pk.ParseFromString(entry)  # one Packet.messages entry parses as a Packet with one message
            assert len(pk.messages) == 1
            mp = pk.messages[0]
            assert (mp.channelId, mp.msgType, mp.broadcast, mp.stubId) == (int(d["channel_id"]), 8, 0, 0)
            cdu = W.ChannelDataUpdateMessage()
            cdu.ParseFromString(mp.msgBody)
            assert cdu.contextConnId == 0 and cdu.data.type_url == W.TYPE_URL
            m = W.TestChannelDataMessage()
            m.ParseFromString(cdu.data.value)
            got.setdefault((int(conn[d["sub"]]), int(d["channel_id"])), []).append(m)
        assert set(got) == set(want)
        for key in want:
            assert sorted(x.SerializeToString(deterministic=True) for x in got[key]) == sorted(x.SerializeToString(deterministic=True) for x in want[key]), key
            n_checked += len(want[key])
        # ---- framed packets per connection
        conn_off = np.zeros(S + 1, np.uint64)
        conn_len = np.zeros(S, np.uint32)
        conn_frames = np.zeros(S, np.uint32)
        out = np.zeros(1 << 23, np.uint8)
        out_len, dropped = C.c_uint64(), C.c_uint32()
        st_ = e.L.chd_frame_packets(e.h, capi.ptr(compression), capi.ptr(conn_off), capi.ptr(conn_len), capi.ptr(conn_frames), capi.ptr(out), out.size,
                                     C.byref(out_len), C.byref(dropped))
        assert st_ == capi.OK, e.L.chd_last_error(e.h)
        assert dropped.value == 0
        for j in range(S):
            buf = bytes(out[int(conn_off[j]):int(conn_off[j]) + int(conn_len[j])])
            pos, msgs, frames = 0, [], 0
            while pos < len(buf):  # connection.go:456-520: tag, size, compression type, body
                assert buf[pos] == 67 and buf[pos + 1] == 72
                size, ct = (buf[pos + 2] << 8) | buf[pos + 3], buf[pos + 4]
                assert ct == compression[j] and size <= 0xFFFF
                body = buf[pos + 5:pos + 5 + size]
                assert len(body) == size
                if ct == 1:
                    body = _snappy_decode(body)
                    assert len(body) <= 0xFFFF
                pk = W.Packet()
                pk.ParseFromString(body)
                msgs += list(pk.messages)
                pos += 5 + size
                frames += 1
            assert frames == conn_frames[j]
            n_multi_frame += frames > 1
            mine = [(int(d["channel_id"]), i) for i, d in enumerate(due) if d["sub"] == j]
            assert len(msgs) == len(mine)
            for mp, (ch, i) in zip(msgs, sorted(mine, key=lambda x: x[1])):  # packet order = ascending due index
                k = int(cls_of[i])
                assert mp.SerializeToString() == W.Packet.FromString(bytes(blob[int(cls_off[k]):int(cls_off[k + 1])])).messages[0].SerializeToString()
    assert n_checked > 300 and n_update_msgs > 100 and n_shared > 20
    e.close()


def _parse_frames(buf):
    """A connection's bytes -> [(compression type, size field, body)], read like connection.go:456-520 reads them."""
    frames, pos = [], 0
    while pos < len(buf):
        assert buf[pos:pos + 2] == b"CH"
        size, ct = (buf[pos + 2] << 8) | buf[pos + 3], buf[pos + 4]
        assert 0 < size <= 0xFFFF and pos + 5 + size <= len(buf)  # a wrapped size field shows up here or as a short parse
        frames.append((ct, size, buf[pos + 5:pos + 5 + size]))
        pos += 5 + size
    assert pos == len(buf)
    return frames


class _Row:
    """A row of 10 x 10 cells.  Connection j subscribes with SpotsAOI (dist 0: a 20 ms interval) to exactly the cells subs[j]
    at t = 0; every pair is subscribed on the oracle's data.go emulation too.  The device treats payload bytes as opaque, so
    tests choose them (random bytes included) to put each layer of the wire format at the size under test."""

    def __init__(self, chd, oracle, n_cells, subs, id_start=S0):
        from tests._oracle import make_grid

        self.chd, self.capi, self.n_cells, self.id_start = chd, chd.capi, n_cells, id_start
        S = len(subs)
        self.conn = np.arange(101, 101 + S, dtype=np.uint32)
        self.e = chd.engine.Engine(chd.engine.grid_cfg(0, 0, 10, 10, n_cells, 1, id_start=id_start), 8, S)
        self.e.set_subscribers(self.conn)
        self.e.set_entities(np.array([5.0]), np.array([5.0]))
        self.e.build()
        n_sp = np.array([len(c) for c in subs], np.uint32)
        off = np.concatenate([[0], np.cumsum(n_sp)]).astype(np.uint32)
        x = np.array([10.0 * c + 5.0 for cs in subs for c in cs])
        batch, keep = chd.engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), kind=np.full(S, self.capi.AOI_SPOTS, np.uint8),
                                            spots=(off, n_sp, x, np.full(len(x), 5.0), np.zeros(len(x), np.uint32)))
        self.e.update_interest(batch, 0)
        og = make_grid(0, 0, 10, 10, n_cells, 1, id_start=id_start)
        self.chans = [oracle.channel() for _ in range(n_cells)]
        for j, cs in enumerate(subs):
            res, st = oracle.query(og, spots=[(10.0 * c + 5.0, 5.0) for c in cs], spot_dists=[0] * len(cs))
            assert st == 0 and res == {id_start + c: 0 for c in cs}
            for c in cs:
                self.chans[c].subscribe(int(self.conn[j]), 0, oracle.damping(0, 20), 0, True, False)
        assert self.e.summary().n_pairs == sum(len(c) for c in subs)
        self.rings = [[] for _ in range(n_cells)]  # (arrival, sender, bytes), cumulative like the reference's update buffer

    def tick(self, t, new_entries, fulls, compression):
        """new_entries: {cell: [(arrival, sender conn id, bytes)]} appended to the rings; fulls: every cell's full data bytes.
        Runs the fan-out, assembles the class entries and frames every connection.  Returns the device's outputs and, per due
        record, the value the oracle's decision selects: the full data (FULL) or the selected ring entries' bytes in ring
        order (UPDATE)."""
        from tests import _wire as W

        capi, e = self.capi, self.e
        for c, ents in new_entries.items():
            for a, snd, b in ents:
                self.rings[c].append((a, snd, b))
                self.chans[c].on_update(a, snd)
        roff = np.concatenate([[0], np.cumsum([len(r) for r in self.rings])]).astype(np.uint32)
        flat = [x for r in self.rings for x in r]
        e.set_rings(roff, np.array([f[0] for f in flat], np.int64), np.array([f[1] for f in flat], np.uint32),
                    np.array([k + 1 for r in self.rings for k in range(len(r))], np.uint64), np.array([len(r) for r in self.rings], np.uint64))
        eoff = np.concatenate([[0], np.cumsum([len(f[2]) for f in flat])]).astype(np.uint64)
        eb = np.frombuffer(b"".join(f[2] for f in flat) or b"\0", np.uint8).copy()
        foff = np.concatenate([[0], np.cumsum([len(b) for b in fulls])]).astype(np.uint64)
        fb = np.frombuffer(b"".join(fulls) or b"\0", np.uint8).copy()
        assert e.L.chd_set_payload_bytes(e.h, capi.ptr(eoff), len(flat), capi.ptr(eb), capi.ptr(foff), capi.ptr(fb), W.TYPE_URL.encode(),
                                         W.MSG_CHANNEL_DATA_UPDATE) == capi.OK
        e.fanout_tick(t)
        n_due = int(e.summary().n_due)
        due = e.get_due(n_due)
        want = {}
        for c in range(self.n_cells):
            for d in self.chans[c].tick_data_ex(t):
                v = fulls[c] if d["kind"] == 0 else b"".join(self.rings[c][p][2] for p in d["selected"])
                want[(d["conn"], self.id_start + c, d["kind"], d["window_hi"])] = (v, d)
        r = dict(due=due, value=[], oracle=[])
        for d in due:
            v, od = want.pop((int(self.conn[d["sub"]]), int(d["channel_id"]), int(d["kind"]), int(d["window_hi"])))
            r["value"].append(v)
            r["oracle"].append(od)
        assert not want, "decisions the device did not make: %s" % sorted(want)
        ncls, blen = C.c_uint32(), C.c_uint64()
        cls_off = np.zeros(n_due + 2, np.uint64)
        blob = np.zeros(1 << 22, np.uint8)
        assert e.L.chd_assemble_payloads(e.h, C.byref(ncls), capi.ptr(cls_off), n_due + 1, capi.ptr(blob), blob.size, C.byref(blen)) == capi.OK
        r["cls_of"], r["cls_rep"], _ = e.due_classes(n_due)
        r["entry"] = [bytes(blob[int(cls_off[k]):int(cls_off[k + 1])]) for k in r["cls_of"].tolist()]
        S = len(self.conn)
        conn_off, conn_len, conn_frames = np.zeros(S + 1, np.uint64), np.zeros(S, np.uint32), np.zeros(S, np.uint32)
        out = np.zeros(1 << 23, np.uint8)
        olen, dropped = C.c_uint64(), C.c_uint32()
        comp = np.ascontiguousarray(compression, np.uint8)
        assert e.L.chd_frame_packets(e.h, capi.ptr(comp), capi.ptr(conn_off), capi.ptr(conn_len), capi.ptr(conn_frames), capi.ptr(out), out.size,
                                     C.byref(olen), C.byref(dropped)) == capi.OK
        assert olen.value == int(conn_off[S])
        r.update(conn_off=conn_off, conn_len=conn_len, conn_frames=conn_frames, dropped=dropped.value,
                 conn_bytes=[bytes(out[int(conn_off[s]):int(conn_off[s]) + int(conn_len[s])]) for s in range(S)])
        return r

    def restated_flush(self, r):
        """Per connection: the restated flush of its class entries in ascending due index -> [(packets, n_dropped)]."""
        from tests import _wire as W

        res = []
        for s in range(len(self.conn)):
            mine = [i for i in range(len(r["due"])) if int(r["due"][i]["sub"]) == s]
            res.append(W.flush([W.Packet.FromString(r["entry"][i]).messages[0] for i in mine]))
        return res


def _value_len(layer, target, ch, n_max=1 << 17):
    """The value length that puts `layer` (value / any / cdu / mp / entry) of a class entry for channel `ch` at exactly
    `target` bytes, measured with the protobuf runtime (every layer grows strictly with the value)."""
    from google.protobuf import any_pb2

    from tests import _wire as W

    def size(n):
        v = b"\0" * n
        a = any_pb2.Any(type_url=W.TYPE_URL, value=v)
        return {"value": n, "any": a.ByteSize(), "cdu": W.ChannelDataUpdateMessage(data=a).ByteSize(),
                "mp": W.message_pack(ch, v).ByteSize(), "entry": len(W.class_entry(ch, v))}[layer]

    lo, hi = 0, n_max
    while lo < hi:
        mid = (lo + hi) // 2
        if size(mid) < target:
            lo = mid + 1
        else:
            hi = mid
    assert size(lo) == target, (layer, target, ch)
    return lo


@pytest.mark.parametrize("id_start", [0, 0x10000, (1 << 21) - 8, (1 << 28) - 8, (1 << 32) - 256])
def test_class_entries_are_the_wire_bytes(chd, oracle, id_start):
    """Every class entry equals, byte for byte, the protobuf runtime's serialization of the Packet entry Send would queue:
    every layer (value, Any, ChannelDataUpdateMessage, MessagePack, entry) at 127 / 128 and 16383 / 16384 bytes, an empty full
    data message, channel ids of every varint width (0 is omitted), multi-entry UPDATE windows, a self-skipped singleton class
    and an UPDATE class shared by two connections.  Tick 1 sends every cell FULL; tick 2 sends UPDATE windows whose entries
    split the same value lengths."""
    from tests import _wire as W

    layers = [(ly, tg) for ly in ("value", "any", "cdu", "mp", "entry") for tg in (127, 128, 16383, 16384)]
    n_cells = len(layers) + 2  # + the empty full data message + the self-skip cell
    empty, selfc = len(layers), len(layers) + 1
    rng = np.random.default_rng(id_start % 1009)
    n = [_value_len(ly, tg, id_start + c) for c, (ly, tg) in enumerate(layers)] + [0, 300]
    every = list(range(n_cells))
    row = _Row(chd, oracle, n_cells, [every, every, [selfc]], id_start=id_start)
    fulls = [rng.bytes(k) for k in n]
    t1 = 100 * MS
    r1 = row.tick(t1, {}, fulls, [0, 0, 0])
    assert len(r1["due"]) == 2 * n_cells + 1 and (r1["due"]["kind"] == 0).all()
    new = {}
    for c in range(len(layers)):  # 1..3 entries per cell splitting the value length
        v = rng.bytes(n[c])
        cuts = sorted(rng.integers(0, n[c] + 1, c % 3).tolist())
        parts = [v[a:b] for a, b in zip([0] + cuts, cuts + [n[c]])]
        new[c] = [(t1 + (k + 1) * MS, 7, p) for k, p in enumerate(parts)]
    mine = rng.bytes(40)
    new[selfc] = [(t1 + 1 * MS, 7, rng.bytes(100)), (t1 + 2 * MS, int(row.conn[2]), mine), (t1 + 3 * MS, 7, rng.bytes(200))]
    r2 = row.tick(t1 + 20 * MS, new, fulls, [0, 0, 0])
    assert (r2["due"]["kind"] == 1).all()
    for r in (r1, r2):
        for i, d in enumerate(r["due"]):
            want = W.class_entry(int(d["channel_id"]), r["value"][i])
            assert r["entry"][i] == want, (i, int(d["channel_id"]), len(r["entry"][i]), len(want))
    # the edges the test is for were reached
    width = lambda ch: sum(ch >= 1 << (7 * k) for k in range(5))  # noqa: E731  (bytes of the channelId varint; 0 = omitted)
    widths = {width(int(d["channel_id"])) for r in (r1, r2) for d in r["due"]}
    assert widths == {0: {0, 1}, 0x10000: {3}, (1 << 21) - 8: {3, 4}, (1 << 28) - 8: {4, 5}, (1 << 32) - 256: {5}}[id_start]
    for r in (r1, r2):
        got_layers = {(ly, tg) for i, (ly, tg) in enumerate(layers)
                      if any(int(d["channel_id"]) == id_start + i and len(r["value"][k]) == n[i] for k, d in enumerate(r["due"]))}
        assert got_layers == set(layers)
    sel = [r2["oracle"][i] for i in range(len(r2["due"]))]
    assert sum(len(d["selected"]) > 1 for d in sel) > 10
    skip = [i for i, d in enumerate(sel) if d["self_skipped"]]
    assert len(skip) == 1 and mine not in r2["value"][skip[0]] and len(r2["value"][skip[0]]) == 300
    assert int(r2["cls_of"][skip[0]]) not in {int(r2["cls_of"][i]) for i in range(len(sel)) if i != skip[0]}
    shared = [i for i, d in enumerate(r2["due"]) if int(d["channel_id"]) == id_start + selfc and not sel[i]["self_skipped"]]
    assert len(shared) == 2 and r2["cls_of"][shared[0]] == r2["cls_of"][shared[1]] and len(r2["value"][shared[0]]) == 340
    assert len(r2["cls_rep"]) < len(r2["due"])
    row.e.close()


def _check_frames(r, s, packets, want_raw_only):
    """Connection s's bytes against its restated packets; returns the compression types seen."""
    buf = r["conn_bytes"][s]
    assert r["conn_len"][s] <= r["conn_off"][s + 1] - r["conn_off"][s]
    frames = _parse_frames(buf)
    assert len(frames) == r["conn_frames"][s] == len(packets), (s, len(frames), len(packets))
    cts = []
    for (ct, size, body), pk in zip(frames, packets):
        assert size == len(body)
        if ct == 1:
            assert not want_raw_only and _snappy_decode(body) == pk
        else:
            assert ct == 0 and body == pk
        cts.append(ct)
    return cts


def test_uncompressed_frames_match_flush(chd, oracle):
    """Framing at the 64 KB edges against the restated Send / flush (tests/_wire.py): one connection per edge.  FULL sends
    only, so each cell's full data sets its entry size.  Cells: 0 small, 1..7 MessagePack 65525..65531, 8 small, 9 entry 30000,
    10..12 entries that total 65534 / 65535 / 65536 with cell 9."""
    from tests import _wire as W

    ch = lambda c: S0 + c  # noqa: E731
    n = [_value_len("entry", 1000, ch(0))] + [_value_len("mp", 65525 + k, ch(1 + k)) for k in range(7)]
    n += [_value_len("entry", 2000, ch(8)), _value_len("entry", 30000, ch(9))]
    n += [_value_len("entry", 65534 + k - 30000, ch(10 + k)) for k in range(3)]
    subs = [[1 + k] for k in range(7)]    # MessagePack 65525 .. 65531 alone
    subs += [[9, 10 + k] for k in range(3)]  # packet totals 65534, 65535, 65536
    subs += [[0, 6, 8]]                    # a dropped message (65530) between two sent ones
    subs += [[6, 7]]                       # every message dropped
    subs += [[0, 5, 8]]                    # 1000 + 65533 + 2000: three packets
    row = _Row(chd, oracle, 13, subs)
    rng = np.random.default_rng(11)
    r = row.tick(100 * MS, {}, [rng.bytes(k) for k in n], np.zeros(len(subs), np.uint8))
    assert (r["due"]["kind"] == 0).all()
    for i, d in enumerate(r["due"]):
        assert r["entry"][i] == W.class_entry(int(d["channel_id"]), r["value"][i])
    assert [int(d["channel_id"]) for d in r["due"] if d["sub"] == 10] == [ch(0), ch(6), ch(8)]  # due order puts the drop mid-list
    want = row.restated_flush(r)
    assert r["dropped"] == sum(dr for _, dr in want)
    for s, (packets, _) in enumerate(want):
        assert r["conn_bytes"][s] == b"".join(W.frame(p) for p in packets), s
        _check_frames(r, s, packets, True)
    assert [len(p) for p, _ in want] == [1] * 5 + [0, 0] + [1, 1, 2] + [1, 0, 3]
    assert [dr for _, dr in want] == [0] * 5 + [1, 1] + [0, 0, 0] + [1, 2, 0]
    assert [len(want[7 + k][0][0]) for k in range(2)] == [65534, 65535]
    row.e.close()


def test_compressed_frames_never_overflow_the_size_field(chd, oracle):
    """Snappy connections with packet bodies of 65000 .. 65535 bytes of repeated text, random bytes and random lowercase
    letters.  Every size field is the body length; a snappy frame decodes to the restated packet; a packet whose encoding
    would not fit the 16-bit size field goes out raw with compression type 0 (up to 56146 bytes the encoding always fits)."""
    single, pair = [65000, 65250, 65500, 65533], [65534, 65535]
    per_kind = len(single) + 1 + len(pair)  # cells of one kind: singles, a 30000-byte entry, its partners
    rng = np.random.default_rng(23)
    kinds = {
        "text": lambda k: (b"position update for entity 12345; " * (k // 34 + 1))[:k],
        "random": lambda k: rng.bytes(k),
        "letters": lambda k: rng.integers(97, 123, k, dtype=np.uint8).tobytes(),
    }
    fulls, subs, kind_of = [], [], []
    for ki, (name, make) in enumerate(kinds.items()):
        base = ki * per_kind
        sizes = single + [30000] + [p - 30000 for p in pair]
        fulls += [make(_value_len("entry", sz, S0 + base + j)) for j, sz in enumerate(sizes)]
        subs += [[base + j] for j in range(len(single))] + [[base + len(single), base + len(single) + 1 + j] for j in range(len(pair))]
        kind_of += [name] * (len(single) + len(pair))
    row = _Row(chd, oracle, 3 * per_kind, subs)
    r = row.tick(100 * MS, {}, fulls, np.ones(len(subs), np.uint8))
    want = row.restated_flush(r)
    assert r["dropped"] == 0
    cts = {}
    for s, (packets, dr) in enumerate(want):
        assert dr == 0 and len(packets) == 1 and 65000 <= len(packets[0]) <= 65535
        for ct, (_, size, body) in zip(_check_frames(r, s, packets, False), _parse_frames(r["conn_bytes"][s])):
            if ct == 0:  # snappy.MaxEncodedLen(n) = 32 + n + n/6 <= 65535 up to n = 56146, and bounds the encoder's output
                assert size > 56146 and 32 + 56146 + 56146 // 6 == 0xFFFF
            cts.setdefault(kind_of[s], []).append(ct)
    assert set(cts["text"]) == {1}
    assert 0 in cts["random"]  # the raw fallback is exercised
    row.e.close()


def test_framing_splits_and_drops(chd):
    """connection.go:626-714 / :73-77 with sizes under control: 3 cells in a row, 4 connections subscribed to all of them.
    FULL sends of 50 KB per cell -> 150 KB per connection -> three packets; then UPDATE windows of 60 KB (cell 0), 30 KB (cell 1)
    and 90 KB (cell 2: >= MaxPacketSize - 5, dropped like queuedMessagePackSender.Send does)."""
    from tests import _wire as W

    capi = chd.capi
    e = chd.engine.Engine(chd.engine.grid_cfg(0, 0, 100, 100, 3, 1), 8, 4)
    conn = np.array([11, 12, 13, 14], np.uint32)
    e.set_subscribers(conn)
    e.set_entities(np.array([50.0]), np.array([50.0]))
    e.build()
    batch, keep = chd.engine.make_batch(4, sphere=(np.full(4, 150.0), np.full(4, 50.0), np.full(4, 140.0)))
    e.update_interest(batch, 0)
    assert e.summary().n_pairs == 12

    def msg(n):
        m = W.TestChannelDataMessage()
        m.text = "x" * n
        return m.SerializeToString()

    def run(t, ring_entries, fulls, compression):
        """ring_entries: per cell list of (arrival, sender, bytes)"""
        roff = np.concatenate([[0], np.cumsum([len(r) for r in ring_entries])]).astype(np.uint32)
        flat = [x for r in ring_entries for x in r]
        e.set_rings(roff, np.array([f[0] for f in flat], np.int64), np.array([f[1] for f in flat], np.uint32),
                    np.arange(1, len(flat) + 1, dtype=np.uint64), np.array([len(r) for r in ring_entries], np.uint64))
        eoff = np.concatenate([[0], np.cumsum([len(f[2]) for f in flat])]).astype(np.uint64)
        eb = np.frombuffer(b"".join(f[2] for f in flat) or b"\0", np.uint8).copy()
        foff = np.concatenate([[0], np.cumsum([len(b) for b in fulls])]).astype(np.uint64)
        fb = np.frombuffer(b"".join(fulls) or b"\0", np.uint8).copy()
        assert e.L.chd_set_payload_bytes(e.h, capi.ptr(eoff), len(flat), capi.ptr(eb), capi.ptr(foff), capi.ptr(fb), W.TYPE_URL.encode(), 8) == capi.OK
        e.fanout_tick(t)
        s = e.summary()
        due = e.get_due(s.n_due)
        ncls, blen = C.c_uint32(), C.c_uint64()
        cls_off = np.zeros(int(s.n_due) + 2, np.uint64)
        blob = np.zeros(1 << 20, np.uint8)
        assert e.L.chd_assemble_payloads(e.h, C.byref(ncls), capi.ptr(cls_off), int(s.n_due) + 1, capi.ptr(blob), blob.size, C.byref(blen)) == capi.OK
        cls_of, _, _ = e.due_classes(int(s.n_due))
        conn_off, conn_len, conn_frames = np.zeros(5, np.uint64), np.zeros(4, np.uint32), np.zeros(4, np.uint32)
        out = np.zeros(1 << 21, np.uint8)
        olen, dropped = C.c_uint64(), C.c_uint32()
        comp = np.array(compression, np.uint8)
        assert e.L.chd_frame_packets(e.h, capi.ptr(comp), capi.ptr(conn_off), capi.ptr(conn_len), capi.ptr(conn_frames), capi.ptr(out), out.size,
                                     C.byref(olen), C.byref(dropped)) == capi.OK
        per_conn, bodies = [], []
        for j in range(4):
            buf = bytes(out[int(conn_off[j]):int(conn_off[j]) + int(conn_len[j])])
            pos, frames, packets = 0, [], []
            while pos < len(buf):
                assert buf[pos:pos + 2] == b"CH" and buf[pos + 4] == comp[j]
                size = (buf[pos + 2] << 8) | buf[pos + 3]
                body = buf[pos + 5:pos + 5 + size]
                if comp[j]:
                    body = _snappy_decode(body)
                pk = W.Packet.FromString(body)
                frames.append([(m.channelId, len(m.msgBody)) for m in pk.messages])
                packets.append(body)
                assert len(body) <= 0xFFFF
                pos += 5 + size
            assert len(frames) == conn_frames[j]
            per_conn.append(frames)
            bodies.append(packets)
        entries = {}  # per connection its class entries in ascending due index
        for i, d in enumerate(due):
            k = int(cls_of[i])
            entries.setdefault(int(d["sub"]), []).append(bytes(blob[int(cls_off[k]):int(cls_off[k + 1])]))
        # the restated Send / flush (tests/_wire.py) over those entries
        want = [W.flush([W.Packet.FromString(b).messages[0] for b in entries.get(j, [])]) for j in range(4)]
        return per_conn, bodies, want, dropped.value, due

    # tick 1: everybody's first fan-out = FULL channel data, 50 KB per cell
    fulls = [msg(50000), msg(50000), msg(50000)]
    per_conn, bodies, want, dropped, due = run(100 * MS, [[], [], []], fulls, [0, 1, 0, 1])
    assert dropped == 0 and len(due) == 12 and (due["kind"] == 0).all()
    for j in range(4):
        assert [len(f) for f in per_conn[j]] == [1, 1, 1]  # 3 x 50 KB cannot share a 64 KB packet
        assert sorted(ch for f in per_conn[j] for ch, _ in f) == [S0, S0 + 1, S0 + 2]
        assert bodies[j] == want[j][0]
    # tick 2: updates at 150 ms fall into the catch-up windows; 60 KB + 30 KB are sent (two packets), 90 KB is dropped
    ring = [[(150 * MS, 7, msg(30000)), (151 * MS, 7, msg(30000))], [(150 * MS, 7, msg(30000))],
            [(150 * MS, 7, msg(30000)), (151 * MS, 7, msg(30000)), (152 * MS, 7, msg(30000))]]
    per_conn, bodies, want, dropped, due = run(200 * MS, ring, fulls, [1, 0, 1, 0])
    assert (due["kind"] == 1).all()
    assert dropped == sum(n for _, n in want) > 0
    for j in range(4):
        assert bodies[j] == want[j][0], (j, per_conn[j])
        assert len(want[j][0]) >= 2
    e.close()
