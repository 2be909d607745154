// chd_payload.cuh — the BYTE half of the fan-out (SURVEY.md §8f rank 1 and 4): for every window class of the tick's due list
// assemble the wire bytes of its CHANNEL_DATA_UPDATE message once, then lay every connection's packet(s) out, framed and
// (optionally) snappy-compressed, ready for conn.Write.
//
// Reference path per (connection, due step): accumulate proto.Merge of the selected ring entries into a scratch message
// (data.go:246-256), anypb.New (data.go:295), proto.Marshal(ChannelDataUpdateMessage) (connection.go:58), proto.Marshal(Packet)
// (connection.go:671), snappy.Encode (:678-681), 5-byte tag (:684-688).
// Here: the host supplies the serialized bytes of every ring entry's updateMsg (and of each channel's full data message for
// FULL sends), or, on byte-carrying device rings (include/chd_gpu_ring_bytes.h), the rings keep each entry's bytes beside it.  Parsing the concatenation of serialized protobuf messages IS merging them (protobuf encoding rule: last scalar
// wins, repeated fields append, embedded messages merge), so the merged payload of a window = the concatenation of its selected
// entries' bytes, wrapped in the fixed field headers of Any / ChannelDataUpdateMessage / MessagePack / Packet:
//   entry  = 0x0A len(mp) mp                                   (Packet.messages, channeld.proto:10-12)
//   mp     = 0x08 channelId  0x20 msgType  0x2A len(cdu) cdu   (MessagePack; broadcast = stubId = 0 are omitted, data.go:301-308)
//   cdu    = 0x0A len(any) any                                 (ChannelDataUpdateMessage.data; contextConnId = 0 omitted)
//   any    = 0x0A len(url) url  0x12 len(value) value          (google.protobuf.Any)
// Like proto3 Marshal, a channelId / msgType of 0 and an empty type_url / value are omitted, so every entry has the size the
// reference's send rules measure.  Valid for channel data types merged by the default reflection merge without merge options
// (data.go:326-388); custom MergeableChannelData types stay on the host.  The wrapper layers are fixed proto3 encodings, so for
// a given `value` the class entry is fully determined and the tests compare it byte for byte with the protobuf runtime's
// serialization.  Only `value` itself (the concatenation of the selected entries) can differ in bytes from what Go would send
// after merging (field order of a merged message, map order); it parses to the same message.  The framing is checked against
// a plain restatement of connection.go's Send / flush rules (tests/_wire.py).
#pragma once
#include "chd_types.cuh"

namespace chd {

constexpr uint32_t PKT_MAX = 0x00ffff;  // MaxPacketSize (connection.go:27)
constexpr uint32_t PKT_HDR = 5;         // PacketHeaderSize (connection.go:28): 'C' 'H' size_hi size_lo compressionType

struct PayloadIn {
    const unsigned long long* entry_off;  // [R+1] byte offsets of the ring entries' serialized updateMsg (ring order of chd_set_rings)
    const uint8_t* entry_bytes;
    const unsigned long long* full_off;   // [C+1] byte offsets of each channel's serialized full data message
    const uint8_t* full_bytes;
    const uint8_t* type_url;              // Any.type_url of the channel data type
    uint32_t url_len;
    uint32_t msg_type;                    // MessageType_CHANNEL_DATA_UPDATE = 8
    // byte-carrying device rings (chd_rings_reserve_bytes) instead of entry_off / entry_bytes, or ring_bytes == nullptr: entry k
    // of cell c is ring_len[k] bytes at ring_bytes + c * bytes_per_cell + ring_pos[k]
    const uint8_t* ring_bytes;
    const uint32_t* ring_pos;
    const uint32_t* ring_len;
    uint64_t bytes_per_cell;
};

struct ByteSpan {
    const uint8_t* p;
    uint64_t n;
};
// the serialized updateMsg of ring entry k of `cell`
__device__ __forceinline__ ByteSpan entry_span(const PayloadIn& in, uint32_t cell, uint32_t k) {
    if (in.ring_bytes) return ByteSpan{in.ring_bytes + cell * in.bytes_per_cell + in.ring_pos[k], in.ring_len[k]};
    return ByteSpan{in.entry_bytes + in.entry_off[k], in.entry_off[k + 1] - in.entry_off[k]};
}

__device__ __forceinline__ uint32_t varint_len(uint64_t v) {
    uint32_t n = 1;
    while (v >= 0x80) { v >>= 7; n++; }
    return n;
}
__device__ __forceinline__ uint8_t* put_varint(uint8_t* p, uint64_t v) {
    while (v >= 0x80) { *p++ = (uint8_t)(v | 0x80); v >>= 7; }
    *p++ = (uint8_t)v;
    return p;
}

struct MsgSizes {
    uint64_t value, any, cdu, mp, entry;
};
// proto3 Marshal omits a scalar field equal to 0 and a bytes / string field that is empty; a set message field (Any inside
// ChannelDataUpdateMessage) is written even when empty
__device__ __forceinline__ uint64_t scalar_field_len(uint64_t v) { return v ? 1 + varint_len(v) : 0; }
__device__ __forceinline__ uint64_t bytes_field_len(uint64_t len) { return len ? 1 + varint_len(len) + len : 0; }
__device__ __forceinline__ MsgSizes msg_sizes(uint64_t value_len, uint32_t url_len, uint32_t channel_id, uint32_t msg_type) {
    MsgSizes s;
    s.value = value_len;
    s.any = bytes_field_len(url_len) + bytes_field_len(value_len);
    s.cdu = 1 + varint_len(s.any) + s.any;
    s.mp = scalar_field_len(channel_id) + scalar_field_len(msg_type) + 1 + varint_len(s.cdu) + s.cdu;
    s.entry = 1 + varint_len(s.mp) + s.mp;
    return s;
}

// The ring entries a decision merges (data.go:226-256), replayed from the decision's identity: FULL -> the channel's data
// message; UPDATE -> entries in insertion order with lastUpdateTime <= arrival <= window_hi, lastUpdateTime starting at `lo`
// and advancing to every picked arrival, own updates skipped when the class is a self-skipped singleton.
template <typename F>
__device__ __forceinline__ void for_each_selected(const RingDev& ring, uint32_t ring_total, uint32_t cell, int64_t lo, int64_t hi, bool skipped,
                                                  uint32_t me, F&& f) {
    const uint32_t r0 = min(ring.off[cell], ring_total), r1 = min(ring.end[cell], ring_total);
    int64_t last_update = lo > 0 ? lo : 0;
    for (uint32_t k = r0; k < r1; k++) {
        const int64_t a = ring.arrival[k];
        if (skipped && ring.sender[k] == me) continue;
        if (a >= last_update && a <= hi) {
            f(k);
            last_update = a;
        }
    }
}

// pass 1: wire size of every class's Packet entry (one thread per class)
__global__ void __launch_bounds__(128)
    payload_size_kernel(uint32_t n_classes, const uint32_t* __restrict__ class_rep, const chd_due* __restrict__ due, const DueKey* __restrict__ key,
                        RingDev ring, const uint32_t* __restrict__ conn_id, PayloadIn in, uint32_t* __restrict__ cls_len,
                        unsigned long long* bump_epoch) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0 && bump_epoch) *bump_epoch = chd_next_epoch(*bump_epoch);
    if (k >= n_classes) return;
    const uint32_t i = class_rep[k];
    const chd_due d = due[i];
    const DueKey dk = key[i];
    const uint32_t cell = (uint32_t)(dk.word >> 34);
    uint64_t value = 0;
    if (d.kind == 0) {
        value = in.full_off[cell + 1] - in.full_off[cell];
    } else {
        const bool skipped = (dk.word >> 32) & 1ull;
        const uint32_t me = skipped ? conn_id[(uint32_t)dk.word] : 0u;
        for_each_selected(ring, *ring.total, cell, dk.lo, d.window_hi, skipped, me,
                          [&](uint32_t e) { value += entry_span(in, cell, e).n; });
    }
    const MsgSizes s = msg_sizes(value, in.url_len, d.channel_id, in.msg_type);
    cls_len[k] = s.entry > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)s.entry;
}

// pass 2: write the entries (one warp per class: lane 0 writes the field headers, all lanes copy payload bytes)
__global__ void __launch_bounds__(128)
    payload_write_kernel(uint32_t n_classes, const uint32_t* __restrict__ class_rep, const chd_due* __restrict__ due, const DueKey* __restrict__ key,
                         RingDev ring, const uint32_t* __restrict__ conn_id, PayloadIn in, const unsigned long long* __restrict__ cls_off,
                         uint8_t* __restrict__ blob, uint64_t blob_cap) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (k >= n_classes) return;
    if (cls_off[n_classes] > blob_cap) return;
    const uint32_t i = class_rep[k];
    const chd_due d = due[i];
    const DueKey dk = key[i];
    const uint32_t cell = (uint32_t)(dk.word >> 34);
    const bool skipped = (dk.word >> 32) & 1ull;
    const uint32_t me = (d.kind && skipped) ? conn_id[(uint32_t)dk.word] : 0u;
    const uint32_t ring_total = *ring.total;
    uint64_t value = 0;
    if (d.kind == 0) value = in.full_off[cell + 1] - in.full_off[cell];
    else for_each_selected(ring, ring_total, cell, dk.lo, d.window_hi, skipped, me, [&](uint32_t e) { value += entry_span(in, cell, e).n; });
    // all lanes copy the url and the value; lane 0 then writes the field headers in front of them (zero / empty fields
    // omitted like msg_sizes counts them).  The entry ends with the url bytes and the value field, so the sizes give the
    // header lengths.
    const MsgSizes s = msg_sizes(value, in.url_len, d.channel_id, in.msg_type);
    const uint64_t value_field = bytes_field_len(s.value);
    uint8_t* const out = blob + cls_off[k];
    uint8_t* const url_at = out + (s.entry - in.url_len - value_field);
    uint8_t* p = url_at;
    for (uint32_t b = lane; b < in.url_len; b += 32) p[b] = in.type_url[b];
    p += in.url_len + (value_field - s.value);
    if (d.kind == 0) {
        const uint8_t* src = in.full_bytes + in.full_off[cell];
        for (uint64_t b = lane; b < value; b += 32) p[b] = src[b];
    } else {
        for_each_selected(ring, ring_total, cell, dk.lo, d.window_hi, skipped, me, [&](uint32_t e) {
            const ByteSpan sp = entry_span(in, cell, e);
            for (uint64_t b = lane; b < sp.n; b += 32) p[b] = sp.p[b];
            p += sp.n;
        });
    }
    if (lane == 0) {
        uint8_t* h = out;
        *h++ = 0x0A; h = put_varint(h, s.mp);
        if (d.channel_id) { *h++ = 0x08; h = put_varint(h, d.channel_id); }
        if (in.msg_type) { *h++ = 0x20; h = put_varint(h, in.msg_type); }
        *h++ = 0x2A; h = put_varint(h, s.cdu);
        *h++ = 0x0A; h = put_varint(h, s.any);
        if (in.url_len) { *h++ = 0x0A; put_varint(h, in.url_len); }
        if (s.value) { h = url_at + in.url_len; *h++ = 0x12; put_varint(h, s.value); }
    }
}

// ---- per-connection framing (connection.go:626-714)

// decisions per connection (subscriber slot); CHD_DUE_VOID holes are skipped
__global__ void __launch_bounds__(256) frame_count_kernel(const chd_due* __restrict__ due, uint32_t n_due, uint32_t n_slots, uint32_t* __restrict__ cnt,
                                                          unsigned long long* bump_epoch) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && bump_epoch) *bump_epoch = chd_next_epoch(*bump_epoch);
    if (i >= n_due) return;
    const chd_due d = due[i];
    if (d.kind != CHD_DUE_VOID && d.sub < n_slots) atomicAdd(&cnt[d.sub], 1u);
}
__global__ void __launch_bounds__(256) frame_fill_kernel(const chd_due* __restrict__ due, uint32_t n_due, uint32_t n_slots, const uint32_t* __restrict__ off,
                                                         uint32_t* __restrict__ cursor, uint32_t* __restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_due) return;
    const chd_due d = due[i];
    if (d.kind != CHD_DUE_VOID && d.sub < n_slots) idx[off[d.sub] + atomicAdd(&cursor[d.sub], 1u)] = i;
}

// snappy.MaxEncodedLen (golang/snappy encode.go): 32 + n + n/6
__host__ __device__ __forceinline__ uint32_t snappy_max_len(uint32_t n) { return 32u + n + n / 6u; }

// Send drops a message whose MessagePack is MaxPacketSize - PacketHeaderSize bytes or longer (connection.go:73-77).  A class
// entry is 0x0A, the MessagePack's length varint and the MessagePack, so its length grows strictly with the MessagePack's:
// the MessagePack reaches the limit exactly when the entry is at least as long as an entry holding a limit-sized MessagePack.
// (Lengths clamped to 0xFFFFFFFF by payload_size_kernel are dropped too.)
constexpr uint32_t MP_DROP = PKT_MAX - PKT_HDR;
__device__ __forceinline__ bool send_drops(uint32_t entry_len) { return entry_len >= 1 + varint_len(MP_DROP) + MP_DROP; }

// Per connection: order its decisions (ascending due index: a deterministic stand-in for the reference's send-queue order,
// which is unspecified across channel goroutines), cut them into packets of at most MaxPacketSize bytes (connection.go:643-659: a
// message that would overflow the packet opens the next one; a message send_drops() refuses is skipped wherever it stands)
// and reserve the connection's output region (worst case for compressed connections).
__global__ void __launch_bounds__(128)
    frame_size_kernel(uint32_t n_slots, const uint32_t* __restrict__ off, uint32_t* __restrict__ idx, const uint32_t* __restrict__ class_of,
                      const uint32_t* __restrict__ cls_len, const uint8_t* __restrict__ compression, uint32_t* __restrict__ conn_cap,
                      uint32_t* __restrict__ n_dropped) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const uint32_t b = off[s], e = off[s + 1];
    for (uint32_t a = b + 1; a < e; a++) {  // insertion sort by due index (lists are a handful of entries)
        const uint32_t v = idx[a];
        uint32_t j = a;
        while (j > b && idx[j - 1] > v) { idx[j] = idx[j - 1]; j--; }
        idx[j] = v;
    }
    const bool comp = compression && compression[s] == 1;
    uint32_t total = 0, cur = 0, dropped = 0;
    for (uint32_t a = b; a < e; a++) {
        const uint32_t L = cls_len[class_of[idx[a]]];
        if (send_drops(L)) { dropped++; continue; }
        if (cur + L > PKT_MAX) {
            total += PKT_HDR + (comp ? snappy_max_len(cur) : cur);
            cur = 0;
        }
        cur += L;
    }
    if (cur) total += PKT_HDR + (comp ? snappy_max_len(cur) : cur);
    conn_cap[s] = total;
    if (dropped) atomicAdd(n_dropped, dropped);
}

// ---- snappy block-format encoder (golang/snappy v0.0.4 is the reference's dependency, go.mod:6; the format — varint length,
// then literal / copy elements — is the public snappy format description).  Greedy matcher over a 4096-entry hash table of
// 4-byte sequences; emits copy-2 elements (1..64 bytes, 16-bit offset) and literals.  Any conforming decoder restores the
// input; the bytes differ from Go's encoder (as Go's differ from C++ snappy's): parity = decode(ours) == input.
constexpr int SNAPPY_HASH_BITS = 12;
__device__ __forceinline__ uint32_t load32u(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint8_t* snappy_emit_literal(uint8_t* op, const uint8_t* lit, uint32_t len) {
    if (len == 0) return op;
    const uint32_t n = len - 1;
    if (n < 60) *op++ = (uint8_t)(n << 2);
    else if (n < 256) { *op++ = 60 << 2; *op++ = (uint8_t)n; }
    else { *op++ = 61 << 2; *op++ = (uint8_t)n; *op++ = (uint8_t)(n >> 8); }  // packets are < 64 KB
    for (uint32_t i = 0; i < len; i++) op[i] = lit[i];
    return op + len;
}
__device__ __forceinline__ uint8_t* snappy_emit_copy(uint8_t* op, uint32_t offset, uint32_t len) {
    while (len > 0) {
        uint32_t l = len > 64 ? 64 : len;
        if (len > 64 && len - 64 < 4) l = 60;  // never leave a tail shorter than 4 (keeps every element a plain copy-2)
        *op++ = (uint8_t)(((l - 1) << 2) | 2);
        *op++ = (uint8_t)offset;
        *op++ = (uint8_t)(offset >> 8);
        len -= l;
    }
    return op;
}
// single-thread encoder; `table` = 1 << SNAPPY_HASH_BITS u16 entries (position + 1, 0 = empty), cleared by the caller
__device__ __forceinline__ uint32_t snappy_encode(const uint8_t* in, uint32_t n, uint8_t* out, uint16_t* table) {
    uint8_t* op = put_varint(out, n);
    uint32_t ip = 0, lit = 0;
    while (ip + 4 <= n) {
        const uint32_t w = load32u(in + ip);
        const uint32_t h = (w * 0x1e35a7bdu) >> (32 - SNAPPY_HASH_BITS);
        const uint32_t cand1 = table[h];
        table[h] = (uint16_t)(ip + 1);
        if (cand1 && load32u(in + cand1 - 1) == w) {
            const uint32_t cand = cand1 - 1;
            op = snappy_emit_literal(op, in + lit, ip - lit);
            uint32_t len = 4;
            while (ip + len < n && in[cand + len] == in[ip + len]) len++;
            op = snappy_emit_copy(op, ip - cand, len);
            ip += len;
            lit = ip;
        } else {
            ip++;
        }
    }
    op = snappy_emit_literal(op, in + lit, n - lit);
    return (uint32_t)(op - out);
}

// pass 2 of the framing: one warp per connection writes its packets back to back into its region: tag + body
// (body = concatenation of its decisions' class entries = a marshalled Packet; snappy-compressed for connections that asked for it).
__global__ void __launch_bounds__(128)
    frame_write_kernel(uint32_t n_slots, const uint32_t* __restrict__ off, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ class_of,
                       const uint32_t* __restrict__ cls_len, const unsigned long long* __restrict__ cls_off, const uint8_t* __restrict__ blob,
                       const uint8_t* __restrict__ compression, const unsigned long long* __restrict__ conn_off, uint8_t* __restrict__ out,
                       uint64_t out_cap, uint8_t* __restrict__ stage, uint32_t* __restrict__ conn_len, uint32_t* __restrict__ conn_frames) {
    __shared__ uint16_t s_table[4][1 << SNAPPY_HASH_BITS];
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (s >= n_slots) return;
    if (conn_off[n_slots] > out_cap) return;
    const uint32_t b = off[s], e = off[s + 1];
    const bool comp = compression && compression[s] == 1;
    uint8_t* region = out + conn_off[s];
    uint8_t* scratch = stage + conn_off[s];  // same offsets: a connection's staging never exceeds its (worst-case) output region
    uint32_t pos = 0, frames = 0;
    uint32_t a = b;
    while (a < e) {
        // one packet: entries a .. a2-1
        uint32_t cur = 0, a2 = a;
        while (a2 < e) {
            const uint32_t L = cls_len[class_of[idx[a2]]];
            if (send_drops(L)) { a2++; if (cur == 0) a = a2; continue; }  // dropped message (skipped wherever it stands)
            if (cur + L > PKT_MAX) break;
            cur += L;
            a2++;
        }
        if (cur == 0) break;
        uint8_t* body = comp ? scratch + pos : region + pos + PKT_HDR;
        uint32_t wpos = 0;
        for (uint32_t k = a; k < a2; k++) {
            const uint32_t c = class_of[idx[k]];
            const uint32_t L = cls_len[c];
            if (send_drops(L)) continue;
            const uint8_t* src = blob + cls_off[c];
            for (uint32_t i = lane; i < L; i += 32) body[wpos + i] = src[i];
            wpos += L;
        }
        __syncwarp();
        uint32_t body_len = cur;
        bool snappy = false;
        if (comp) {
            for (int i = lane; i < (1 << SNAPPY_HASH_BITS); i += 32) s_table[w][i] = 0;
            __syncwarp();
            if (lane == 0) body_len = snappy_encode(body, cur, region + pos + PKT_HDR, s_table[w]);
            body_len = __shfl_sync(0xffffffffu, body_len, 0);
            snappy = body_len <= PKT_MAX;
            if (!snappy) {  // encoded body overflows the 16-bit size field: send the packet raw (chd_gpu.h, chd_frame_packets)
                __syncwarp();
                for (uint32_t i = lane; i < cur; i += 32) region[pos + PKT_HDR + i] = body[i];
                body_len = cur;
            }
        }
        if (lane == 0) {  // 'C' 'H' size_hi size_lo compressionType (connection.go:684-688)
            uint8_t* t = region + pos;
            t[0] = 67; t[1] = 72; t[2] = (uint8_t)((body_len >> 8) & 0xff); t[3] = (uint8_t)(body_len & 0xff); t[4] = snappy ? 1 : 0;
        }
        pos += PKT_HDR + body_len;
        frames++;
        a = a2;
    }
    if (lane == 0) {
        conn_len[s] = pos;
        conn_frames[s] = frames;
    }
}

}  // namespace chd
