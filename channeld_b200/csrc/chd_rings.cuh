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
    const uint32_t base = c * cap;
    uint32_t b = begin[c], e = end[c];
    uint64_t mi = msg_index[c];
    const int64_t max_ns = (int64_t)max_interval_ms[c] * 1000000ll;
    for (uint32_t k = u0; k < u1; k++) {
        if (e == base + cap) {  // tail at the end of the slab: slide the live entries to its start
            uint32_t n = e - b;
            if (n == cap) {  // no room at all: the oldest entry is dropped (capacity too small for the reference's unbounded list)
                atomicOr(overflow, (uint32_t)CHD_OVF_RING);
                b++;
                n--;
            }
#pragma unroll 1  // (unrolled, ptxas spills 16 bytes of this kernel to the stack)
            for (uint32_t i = 0; i < n; i++) {
                arrival[base + i] = arrival[b + i];
                sender[base + i] = sender[b + i];
                index[base + i] = index[b + i];
            }
            b = base;
            e = base + n;
        }
        const int64_t t = upd_arrival[k];
        mi++;
        arrival[e] = t;
        sender[e] = upd_sender[k];
        index[e] = mi;
        e++;
        if (e - b > RING_MAX_BUFFER && arrival[b] + max_ns < t) b++;  // data.go:166-172
    }
    begin[c] = b;
    end[c] = e;
    msg_index[c] = mi;
}

__global__ void __launch_bounds__(128) ring_len_kernel(uint32_t cells, const uint32_t* __restrict__ begin, const uint32_t* __restrict__ end,
                                                       uint32_t* __restrict__ len) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < cells) len[c] = end[c] - begin[c];
}

// chd_get_rings: live lengths (scanned into a CSR by the caller) and the compacted copy
struct RingLenIn {
    const uint32_t *begin, *end;
    __device__ __forceinline__ uint64_t operator()(uint64_t c) const { return end[c] - begin[c]; }
};
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

}  // namespace chd
