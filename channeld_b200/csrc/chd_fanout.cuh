// chd_fanout.cuh — Channel.tickData (data.go:175-291) for ALL spatial channels in one launch: one thread per
// (subscriber, cell) subscription pair runs the reference's per-connection state machine
//   while t >= lastFanOutTime + interval:           (the queue re-sort at data.go:270-286 re-visits a
//       first time  -> FULL, last = t                connection until it is no longer due: an effective loop)
//       otherwise   -> scan the cell's update ring in insertion order, select entries with
//                      lastUpdateTime <= arrival <= nextFanOutTime (skipping own updates), lastUpdateTime
//                      advancing to every picked arrival; last += interval
// One launch: see fanout_kernel below.
#pragma once
#include "chd_types.cuh"

namespace chd {

__device__ __forceinline__ DueKey make_due_key(uint32_t cell, uint32_t kind, bool skipped, uint32_t sub, int64_t lo) {
    return DueKey{kind ? lo : 0ll, ((uint64_t)cell << 34) | ((uint64_t)kind << 33) | ((uint64_t)(skipped ? 1u : 0u) << 32) | (skipped ? sub : 0u)};
}

constexpr uint32_t FANOUT_MAX_STEPS = 1u << 16;
constexpr uint32_t FANOUT_SLOTS = 2;            // decisions per pair kept by the evaluation pass

// The per-pair state machine of tickData.  Decisions are handed to `emit(j, decision, skipped)`; skipped = an own update
// fell into the decision's window and was left out.  (The window's lower end is window_hi - interval: not passed.)
// Returns the number of decisions; the final state is left in (last, flags, last_index).
// Where the ring entries are read from: global memory, or the block's shared-memory copy of the span its pairs' cells cover.
struct RingGlobal {
    const int64_t* __restrict__ arr;
    const uint32_t* __restrict__ snd;
    const uint64_t* __restrict__ idx;
    __device__ __forceinline__ int64_t arrival(uint32_t k) const { return arr[k]; }
    __device__ __forceinline__ uint32_t sender(uint32_t k) const { return snd[k]; }
    __device__ __forceinline__ uint64_t index(uint32_t k) const { return idx[k]; }
};
struct RingShared {
    const int64_t* arr;  // shared memory
    const uint32_t* snd;
    const uint64_t* idx;
    uint32_t first;  // global index of the first staged entry
    __device__ __forceinline__ int64_t arrival(uint32_t k) const { return arr[k - first]; }
    __device__ __forceinline__ uint32_t sender(uint32_t k) const { return snd[k - first]; }
    __device__ __forceinline__ uint64_t index(uint32_t k) const { return idx[k - first]; }
};

template <typename Ring, typename Emit>
__device__ __forceinline__ uint32_t fanout_eval(const RingDev& ring, const Ring& rg, uint32_t ring_total, int64_t t, uint32_t interval, uint32_t c, uint32_t s,
                                                uint32_t me, uint32_t id_start, int64_t& last, uint8_t& flags, uint64_t& last_index, Emit&& emit) {
    const int64_t step_ns = (int64_t)interval * 1000000ll;  // ChannelTime.AddMs (channel.go:30-32)
    const bool skip_self = flags & PF_SKIP_SELF;
    const uint32_t r0 = min(ring.off[c], ring_total), r1 = min(ring.end[c], ring_total);
    const uint32_t max_steps = interval ? FANOUT_MAX_STEPS : 1u;  // interval 0: the reference never terminates
    uint32_t n_out = 0;
    for (uint32_t step = 0; step < max_steps; step++) {
        const int64_t next = last + step_ns;  // data.go:205
        if (t < next) break;
        int64_t latest = next;
        if (!(flags & PF_HAD_FIRST)) {  // data.go:218-224: whole channel data
            flags |= PF_HAD_FIRST;
            last_index = ring.channel_msg_index ? ring.channel_msg_index[c] : 0ull;
            latest = t;
            chd_due d;
            d.sub = s; d.channel_id = c + id_start; d.kind = 0; d.n_selected = 0; d.first_sel = 0; d.last_sel = 0;
            d.sel_hash = 0; d.last_message_index = last_index; d.window_hi = next;
            emit(n_out, d, false);
            n_out++;
        } else if (r1 > r0) {  // data.go:225-265
            int64_t last_update = 0;
            if (last >= last_update) last_update = last;
            uint32_t nsel = 0, first = 0, lastsel = 0;
            uint64_t hash = 0;
            bool skipped = false;  // an own update fell into the window and was left out (data.go:239-242)
            for (uint32_t k = r0; k < r1; k++) {
                const int64_t a = rg.arrival(k);
                if (skip_self && rg.sender(k) == me) {
                    skipped |= a >= last_update && a <= next;
                    continue;
                }
                if (a >= last_update && a <= next) {
                    if (!nsel) first = k - r0;
                    lastsel = k - r0;
                    nsel++;
                    const uint64_t mi = rg.index(k);
                    hash += mi;
                    last_update = a;
                    last_index = mi;
                }
            }
            if (nsel) {
                chd_due d;
                d.sub = s; d.channel_id = c + id_start; d.kind = 1; d.n_selected = nsel; d.first_sel = first; d.last_sel = lastsel;
                d.sel_hash = hash; d.last_message_index = last_index; d.window_hi = next;
                emit(n_out, d, skipped);
                n_out++;
            }
        }
        last = latest;  // data.go:268
    }
    return n_out;
}

// ONE kernel per tick.  Every thread evaluates one pair (state machine once, up to FANOUT_SLOTS decisions kept in
// registers), a block-wide scan turns the decision counts into offsets, one atomicAdd per block reserves the block's
// range of the due list (the running total doubles as n_due), then the decisions are written and the state committed.
// Pairs with more decisions (several intervals behind) re-evaluate from their saved state while writing.
// Pairs are visited grouped by cell (ascending), so the 128 pairs of a block iteration touch the rings of one or two cells:
// the block copies that span of the ring arrays into shared memory once (FANOUT_STAGE entries; wider spans are read from
// global memory) and every thread's window scan runs out of it — the scan is a chain of dependent compares over <= 64
// entries per interval step, i.e. bound by load latency, not by bandwidth.
// The due list is therefore grouped by block and unordered across blocks: it is a SET of send decisions (the
// reference issues them from independent per-channel goroutines, i.e. in no global order either).
constexpr uint32_t FANOUT_STAGE = 640;  // 12.5 KB of shared memory per block

__global__ void __launch_bounds__(128, 8)  // <= 64 registers = 8192 per CTA: a fan-out CTA fits the slot ONE retiring emit CTA (256 x 40) frees
    fanout_kernel(const uint32_t* __restrict__ n_pairs_ptr, uint64_t pair_cap, PairBuf pb, const uint32_t* __restrict__ conn_id, RingDev ring,
                  const int64_t* __restrict__ t_ptr, uint32_t id_start, const uint32_t* __restrict__ by_cell, chd_due* __restrict__ due,
                  DueKey* __restrict__ due_key, uint32_t due_cap, Counters* __restrict__ ctr) {
    __shared__ uint32_t s_warp[4], s_base, s_clo, s_chi;
    __shared__ int64_t s_arr[FANOUT_STAGE];
    __shared__ uint64_t s_idx[FANOUT_STAGE];
    __shared__ uint32_t s_snd[FANOUT_STAGE];
    const uint64_t n = min((uint64_t)*n_pairs_ptr, pair_cap);
    const int64_t t = *t_ptr;  // device-resident so the launch can be replayed from a CUDA graph
    const uint32_t ring_total = *ring.total;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const RingGlobal rglob{ring.arrival, ring.sender, ring.index};
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        uint32_t n_out = 0, interval = 0, c = 0, s = 0, me = 0;
        uint64_t p = 0, last_index0 = 0, last_index = 0;
        int64_t last0 = 0, last = 0;
        uint8_t flags0 = 0, flags = 0;
        chd_due d0, d1;
        bool sk0 = false, sk1 = false, due_now = false;
        int64_t tc = t;  // ChannelTime of this pair's channel: every channel counts from its own start (channel.go:178)
        if (i < n) {
            p = by_cell[i];
            interval = pb.interval[p];
            last0 = last = pb.last[p];
            c = pb.cell[p];
            if (ring.start) tc = t - ring.start[c];
            due_now = tc >= last + (int64_t)interval * 1000000ll;  // (else: the common cheap exit, no further state is read)
            if (threadIdx.x == 0) s_clo = c;
            if (i + 1 == n || threadIdx.x == blockDim.x - 1) s_chi = c;
        }
        __syncthreads();  // also: the previous iteration's readers of the staged span / s_warp / s_base are done
        // the ring entries of cells s_clo .. s_chi (ascending cells: ascending, disjoint entry ranges)
        const uint32_t span0 = min(ring.off[s_clo], ring_total), span1 = min(ring.end[s_chi], ring_total);
        const bool staged = span1 >= span0 && span1 - span0 <= FANOUT_STAGE;
        if (staged) {
            for (uint32_t k = span0 + threadIdx.x; k < span1; k += blockDim.x) {
                s_arr[k - span0] = ring.arrival[k];
                s_snd[k - span0] = ring.sender[k];
                s_idx[k - span0] = ring.index[k];
            }
        }
        __syncthreads();
        const RingShared rsh{s_arr, s_snd, s_idx, span0};
        if (due_now) {
            flags0 = flags = pb.flags[p];
            last_index0 = last_index = pb.last_index[p];
            s = pb.sub[p];
            me = conn_id[s];
            auto keep = [&](uint32_t j, const chd_due& d, bool skipped) {
                if (j == 0) { d0 = d; sk0 = skipped; }
                else if (j == 1) { d1 = d; sk1 = skipped; }
            };
            n_out = staged ? fanout_eval(ring, rsh, ring_total, tc, interval, c, s, me, id_start, last, flags, last_index, keep)
                           : fanout_eval(ring, rglob, ring_total, tc, interval, c, s, me, id_start, last, flags, last_index, keep);
        }
        // block-wide exclusive offsets of n_out (128 threads = 4 warps)
        uint32_t incl = n_out;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t a = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += a;
        }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        uint32_t off = incl - n_out;
        for (int k = 0; k < w; k++) off += s_warp[k];
        if (threadIdx.x == 0) {
            const uint32_t total = s_warp[0] + s_warp[1] + s_warp[2] + s_warp[3];
            s_base = total ? atomicAdd(&ctr->n_due, total) : 0u;
        }
        __syncthreads();
        // Transactional capacity rule: a pair whose decisions do not fit the due list is left exactly as it was (nothing
        // written, no state committed): it is still due at the next tick and catches up then (CHD_OVF_DUE is raised,
        // n_due = the capacity that would have been needed).
        bool fits = true;
        if (n_out) {
            const uint32_t o = s_base + off;
            const int64_t step_ns = (int64_t)interval * 1000000ll;  // an UPDATE decision's window starts at window_hi - interval
            fits = (uint64_t)o + n_out <= due_cap;
            if (!fits) {
                atomicOr(&ctr->overflow, (uint32_t)CHD_OVF_DUE);
                for (uint32_t j = 0; j < n_out && (uint64_t)o + j < due_cap; j++) due[o + j].kind = CHD_DUE_VOID;  // a hole, not a decision
            } else if (n_out <= FANOUT_SLOTS) {
                due[o] = d0; due_key[o] = make_due_key(c, d0.kind, sk0, s, d0.window_hi - step_ns);
                if (n_out > 1) { due[o + 1] = d1; due_key[o + 1] = make_due_key(c, d1.kind, sk1, s, d1.window_hi - step_ns); }
            } else {  // several intervals behind: re-evaluate from the saved state, writing directly
                last = last0; flags = flags0; last_index = last_index0;
                auto put = [&](uint32_t j, const chd_due& d, bool skipped) {
                    due[o + j] = d; due_key[o + j] = make_due_key(c, d.kind, skipped, s, d.window_hi - step_ns);
                };
                if (staged) fanout_eval(ring, rsh, ring_total, tc, interval, c, s, me, id_start, last, flags, last_index, put);
                else fanout_eval(ring, rglob, ring_total, tc, interval, c, s, me, id_start, last, flags, last_index, put);
            }
        }
        if (i < n && fits && (n_out || last != last0)) {  // commit (steps without a decision still advance lastFanOutTime)
            pb.last[p] = last;
            pb.flags[p] = flags;
            pb.last_index[p] = last_index;
        }
    }
}

}  // namespace chd
