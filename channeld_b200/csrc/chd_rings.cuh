// chd_rings.cuh — ChannelData.OnUpdate's buffer maintenance on the device (data.go:149-173), for every spatial channel at once:
//   d.msgIndex++ ; push (arrivalTime, senderConnId, messageIndex) ; if len > MaxUpdateMsgBufferSize (512) and the OLDEST entry
//   is older than maxFanOutIntervalMs it is removed (one removal per append: the buffer may stay longer than 512).
// The opaque half of OnUpdate (merging the update into the channel's data message) stays with the host.
// Storage: each cell owns a slab of `cap` entries inside the ring arrays; [begin, end) is the live ring in insertion order; when
// the tail reaches the end of the slab the live entries slide back to its start.  A slab that is completely full of live
// entries drops its oldest one (CHD_OVF_RING is raised: give the rings a larger capacity).
#pragma once
#include "chd_types.cuh"

namespace chd {

constexpr uint32_t RING_MAX_BUFFER = 512;  // MaxUpdateMsgBufferSize, data.go:53-55

__global__ void __launch_bounds__(128)
    rings_init_kernel(uint32_t cells, uint32_t cap, uint32_t* __restrict__ begin, uint32_t* __restrict__ end) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c <= cells) begin[c] = end[c] = min(c, cells) * cap;  // ([cells]: sentinel)
}

// One cell's walk over its updates of one append, in the order given: the rule above, written once for both append kernels.  The
// hooks `h` own the storage: drop() raises CHD_OVF_RING as a full entry slab loses its oldest entry b; slide(base, b, n) moves
// entries [b, b + n) to the slab start; make_room(k, b, e) runs before update k is pushed and may drop oldest entries (b advances);
// push(e, k, t, mi) writes entry e; evict(b) runs as the 512 rule removes entry b.  `arrival` is what push writes (read back by
// the 512 rule).  Every value the walk computes is the same in each thread that runs it.
template <typename H>
__device__ __forceinline__ void ring_walk(uint32_t base, uint32_t cap, uint32_t u0, uint32_t u1, const int64_t* __restrict__ upd_arrival,
                                          const int64_t* arrival, int64_t max_ns, uint32_t& b, uint32_t& e, uint64_t& mi, H& h) {
    for (uint32_t k = u0; k < u1; k++) {
        if (e == base + cap) {  // tail at the end of the slab: slide the live entries to its start
            uint32_t n = e - b;
            if (n == cap) {  // no room at all: the oldest entry is dropped (capacity too small for the reference's unbounded list)
                h.drop(b);
                b++;
                n--;
            }
            h.slide(base, b, n);
            b = base;
            e = base + n;
        }
        const int64_t t = upd_arrival[k];
        h.make_room(k, b, e);
        mi++;
        h.push(e, k, t, mi);
        e++;
        if (e - b > RING_MAX_BUFFER && arrival[b] + max_ns < t) {  // data.go:166-172
            h.evict(b);
            b++;
        }
    }
}

// the entry metadata of rings_append_kernel (one thread per cell)
struct RingSlots {
    int64_t* __restrict__ arrival;
    uint32_t* __restrict__ sender;
    uint64_t* __restrict__ index;
    const uint32_t* __restrict__ upd_sender;
    uint32_t* overflow;
    __device__ __forceinline__ void drop(uint32_t) const { atomicOr(overflow, (uint32_t)CHD_OVF_RING); }
    __device__ __forceinline__ void slide(uint32_t base, uint32_t b, uint32_t n) const {
#pragma unroll 1  // (unrolled, ptxas spills 16 bytes of this kernel to the stack)
        for (uint32_t i = 0; i < n; i++) {
            arrival[base + i] = arrival[b + i];
            sender[base + i] = sender[b + i];
            index[base + i] = index[b + i];
        }
    }
    __device__ __forceinline__ void make_room(uint32_t, uint32_t&, uint32_t) const {}
    __device__ __forceinline__ void push(uint32_t e, uint32_t k, int64_t t, uint64_t mi) const {
        arrival[e] = t;
        sender[e] = upd_sender[k];
        index[e] = mi;
    }
    __device__ __forceinline__ void evict(uint32_t) const {}
};

// one thread per cell applies the cell's updates of this tick in the order given (upd_off: CSR by cell, clamped to n_updates: a
// lying caller cannot make it read past the uploaded updates)
__global__ void __launch_bounds__(128)
    rings_append_kernel(uint32_t cells, uint32_t cap, const uint32_t* __restrict__ upd_off, uint32_t n_updates, const int64_t* __restrict__ upd_arrival,
                        const uint32_t* __restrict__ upd_sender, uint32_t* __restrict__ begin, uint32_t* __restrict__ end, int64_t* __restrict__ arrival,
                        uint32_t* __restrict__ sender, uint64_t* __restrict__ index, uint64_t* __restrict__ msg_index,
                        const uint32_t* __restrict__ max_interval_ms, uint32_t* __restrict__ overflow) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cells) return;
    const uint32_t u0 = min(upd_off[c], n_updates), u1 = min(upd_off[c + 1], n_updates);
    if (u0 >= u1) return;
    uint32_t b = begin[c], e = end[c];
    uint64_t mi = msg_index[c];
    RingSlots h{arrival, sender, index, upd_sender, overflow};
    ring_walk(c * cap, cap, u0, u1, upd_arrival, arrival, (int64_t)max_interval_ms[c] * 1000000ll, b, e, mi, h);
    begin[c] = b;
    end[c] = e;
    msg_index[c] = mi;
}

// ---- byte-carrying rings (include/chd_gpu_ring_bytes.h): each cell also owns a slab of `bcap` bytes holding the serialized
// updateMsg of its live entries in entry order, [bb, be) relative to the slab; entry slot i carries its position pos[i] (relative
// to the slab) and length len[i].  Per update of L bytes, after the entry slab's rule: while the live bytes + L exceed the slab,
// the oldest entry goes, metadata and bytes (CHD_OVF_RING, like a full entry slab); then, if the tail has no room for L bytes, the
// live bytes slide to the slab start.  The 512 rule releases the bytes of the entry it evicts.  Without CHD_OVF_RING the metadata
// is exactly that of rings_append_kernel.

// moves n elements of each array from src to dst < src, in chunks of 32 per warp: a chunk is read whole before it is written, so a
// shift shorter than the chunk is safe, and a chunk's writes end below the next chunk's reads
template <typename T0, typename T1, typename T2, typename T3, typename T4>
__device__ __forceinline__ void warp_move_down(uint32_t dst, uint32_t src, uint32_t n, int lane, T0* a0, T1* a1, T2* a2, T3* a3, T4* a4) {
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
        const uint32_t i = i0 + lane;
        const bool on = i < n;
        T0 v0{}; T1 v1{}; T2 v2{}; T3 v3{}; T4 v4{};
        if (on) { v0 = a0[src + i]; v1 = a1[src + i]; v2 = a2[src + i]; v3 = a3[src + i]; v4 = a4[src + i]; }
        __syncwarp();
        if (on) { a0[dst + i] = v0; a1[dst + i] = v1; a2[dst + i] = v2; a3[dst + i] = v3; a4[dst + i] = v4; }
    }
    __syncwarp();
}

constexpr uint32_t RING_BYTE_CHUNK = 8;  // bytes per lane and chunk of a byte slide

struct ByteSlots {
    int64_t* arrival;
    uint32_t* sender;
    uint64_t* index;
    uint32_t* pos;
    uint32_t* len;
    const uint32_t* __restrict__ upd_sender;
    const unsigned long long* __restrict__ upd_boff;
    const uint8_t* __restrict__ upd_bytes;
    uint8_t* slab;  // this cell's byte slab
    uint32_t bcap, bb, be;
    uint32_t* overflow;
    int lane;
    __device__ __forceinline__ void drop(uint32_t b) {
        if (lane == 0) atomicOr(overflow, (uint32_t)CHD_OVF_RING);
        bb += len[b];
    }
    __device__ __forceinline__ void slide(uint32_t base, uint32_t b, uint32_t n) { warp_move_down(base, b, n, lane, arrival, sender, index, pos, len); }
    __device__ __forceinline__ void make_room(uint32_t k, uint32_t& b, uint32_t e) {
        const uint32_t L = (uint32_t)(upd_boff[k + 1] - upd_boff[k]);
        while (be - bb + L > bcap && b < e) {  // the byte slab cannot take L more bytes: the oldest entry goes
            drop(b);
            b++;
        }
        if (be + L <= bcap) return;
        // the tail has no room: slide the live bytes to the slab start (bb > 0 here) and rebase the live entries' positions
        const uint32_t n = be - bb, step = 32 * RING_BYTE_CHUNK;
        for (uint32_t i0 = 0; i0 < n; i0 += step) {
            uint8_t v[RING_BYTE_CHUNK];
#pragma unroll
            for (uint32_t j = 0; j < RING_BYTE_CHUNK; j++) {
                const uint32_t i = i0 + j * 32 + lane;
                v[j] = i < n ? slab[bb + i] : 0;
            }
            __syncwarp();
#pragma unroll
            for (uint32_t j = 0; j < RING_BYTE_CHUNK; j++) {
                const uint32_t i = i0 + j * 32 + lane;
                if (i < n) slab[i] = v[j];
            }
        }
        for (uint32_t i = b + lane; i < e; i += 32) pos[i] -= bb;
        __syncwarp();
        be = n;
        bb = 0;
    }
    __device__ __forceinline__ void push(uint32_t e, uint32_t k, int64_t t, uint64_t mi) {
        const uint64_t o = upd_boff[k];
        const uint32_t L = (uint32_t)(upd_boff[k + 1] - o);
        for (uint32_t i = lane; i < L; i += 32) slab[be + i] = upd_bytes[o + i];
        if (lane == 0) {
            arrival[e] = t;
            sender[e] = upd_sender[k];
            index[e] = mi;
            pos[e] = be;
            len[e] = L;
        }
        be += L;
        __syncwarp();
    }
    __device__ __forceinline__ void evict(uint32_t b) { bb += len[b]; }
};

// one warp per cell with updates; the walk is the same in every lane, lane 0 writes the pushed entries and the cursors, all lanes
// move slides and copy bytes.  bcur: [2C] (bb, be) per cell.  upd_boff: [n_updates + 1] byte offsets of the updates in upd_bytes.
__global__ void __launch_bounds__(128)
    rings_append_bytes_kernel(uint32_t cells, uint32_t cap, const uint32_t* __restrict__ upd_off, uint32_t n_updates,
                              const int64_t* __restrict__ upd_arrival, const uint32_t* __restrict__ upd_sender,
                              const unsigned long long* __restrict__ upd_boff, const uint8_t* __restrict__ upd_bytes, uint32_t* __restrict__ begin,
                              uint32_t* __restrict__ end, int64_t* arrival, uint32_t* sender, uint64_t* index, uint32_t* pos, uint32_t* len,
                              uint8_t* slabs, uint32_t bcap, uint32_t* __restrict__ bcur, uint64_t* __restrict__ msg_index,
                              const uint32_t* __restrict__ max_interval_ms, uint32_t* __restrict__ overflow) {
    const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (c >= cells) return;
    const uint32_t u0 = min(upd_off[c], n_updates), u1 = min(upd_off[c + 1], n_updates);
    if (u0 >= u1) return;
    uint32_t b = begin[c], e = end[c];
    uint64_t mi = msg_index[c];
    ByteSlots h{arrival, sender, index, pos, len, upd_sender, upd_boff, upd_bytes, slabs + (uint64_t)c * bcap, bcap, bcur[2 * c], bcur[2 * c + 1],
                overflow, lane};
    ring_walk(c * cap, cap, u0, u1, upd_arrival, arrival, (int64_t)max_interval_ms[c] * 1000000ll, b, e, mi, h);
    if (lane == 0) {
        begin[c] = b;
        end[c] = e;
        msg_index[c] = mi;
        bcur[2 * c] = h.bb;
        bcur[2 * c + 1] = h.be;
    }
}

// chd_get_rings: live lengths (scanned into a CSR by the caller) and the compacted copy
__global__ void __launch_bounds__(128) ring_len_kernel(uint32_t cells, const uint32_t* __restrict__ begin, const uint32_t* __restrict__ end,
                                                       uint32_t* __restrict__ len) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < cells) len[c] = end[c] - begin[c];
}
__global__ void __launch_bounds__(128)
    rings_gather_kernel(uint32_t cells, const uint32_t* __restrict__ begin, const uint32_t* __restrict__ end, const uint32_t* __restrict__ out_off,
                        const int64_t* __restrict__ arrival, const uint32_t* __restrict__ sender, const uint64_t* __restrict__ index,
                        int64_t* __restrict__ o_arrival, uint32_t* __restrict__ o_sender, uint64_t* __restrict__ o_index, uint32_t out_cap) {
    const uint32_t c = blockIdx.x;
    if (c >= cells) return;
    const uint32_t b = begin[c], n = end[c] - b, o = out_off[c];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        if (o + i >= out_cap) break;
        o_arrival[o + i] = arrival[b + i];
        o_sender[o + i] = sender[b + i];
        o_index[o + i] = index[b + i];
    }
}

// chd_get_ring_bytes: per cell its live bytes; then, with the entry CSR (out_off) and the cells' byte offsets (cell_boff), every
// live entry's byte offset and the bytes themselves, compacted (one block per cell)
__global__ void __launch_bounds__(128) ring_bytes_len_kernel(uint32_t cells, const uint32_t* __restrict__ bcur, uint32_t* __restrict__ len) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < cells) len[c] = bcur[2 * c + 1] - bcur[2 * c];
}
__global__ void __launch_bounds__(128)
    ring_bytes_gather_kernel(uint32_t cells, const uint32_t* __restrict__ begin, const uint32_t* __restrict__ end, const uint32_t* __restrict__ out_off,
                             const uint32_t* __restrict__ pos, const uint32_t* __restrict__ bcur, const unsigned long long* __restrict__ cell_boff,
                             const uint8_t* __restrict__ slabs, uint32_t bcap, unsigned long long* __restrict__ o_boff, uint8_t* __restrict__ o_bytes) {
    const uint32_t c = blockIdx.x;
    if (c >= cells) return;
    const uint32_t b = begin[c], n = end[c] - b, o = out_off[c], bb = bcur[2 * c], nb = bcur[2 * c + 1] - bb;
    const unsigned long long ob = cell_boff[c];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) o_boff[o + i] = ob + (pos[b + i] - bb);
    const uint8_t* src = slabs + (uint64_t)c * bcap + bb;
    for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) o_bytes[ob + i] = src[i];
}

}  // namespace chd
