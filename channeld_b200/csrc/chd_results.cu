// chd_results.cu — results: getters, the one-call read-back of a tick (chd_fetch_results), device views.
#include "chd_engine.h"

#include "chd_misc.cuh"

// ---- asynchronous read-back (chd_fetch_results_async): result lists are written straight into the caller's PINNED host buffers by
// a copy kernel that knows the exact list lengths on the device (no host round trip to size a cudaMemcpy), so the host can
// enqueue the next tick before it looks at this one's results.
namespace {
struct PackSeg {
    const void* src;
    void* dst;
    const void* count_ptr;  // device address of the element count (nullptr: `fixed`)
    uint64_t fixed, cap;    // fixed count / capacity of dst in elements
    uint32_t elem_words;    // element size in 32-bit words
    uint32_t count_is_u64;
};
struct PackArgs {
    PackSeg seg[16];  // the most one launch takes: phase A's hop 1, its 14 lists and 2 snapshots of their counts
    int n;
    uint32_t* truncated;  // pinned: set to 1 if a list did not fit its buffer
};
// One segment per blockIdx.y: its count, clamped to the capacity, in 16-byte vectors (full PCIe write bursts) once the destination
// is 16-byte aligned (when the source is aligned the same way), with a scalar head and tail.  Streaming loads and stores: the data is read once and should
// not evict what the emit kernel beside it keeps in L2.
constexpr unsigned COPY_THREADS = 256;
__device__ __forceinline__ void copy_segment(const PackArgs& a) {
    const PackSeg sg = a.seg[blockIdx.y];
    uint64_t n = sg.fixed;
    if (sg.count_ptr) n = sg.count_is_u64 ? *reinterpret_cast<const unsigned long long*>(sg.count_ptr) : (uint64_t)*reinterpret_cast<const uint32_t*>(sg.count_ptr);
    if (n > sg.cap) {
        if (blockIdx.x == 0 && threadIdx.x == 0) *a.truncated = 1;
        n = sg.cap;
    }
    const uint64_t words = n * sg.elem_words;
    const uint32_t* __restrict__ s = reinterpret_cast<const uint32_t*>(sg.src);
    uint32_t* __restrict__ d = reinterpret_cast<uint32_t*>(sg.dst);
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (uint64_t)gridDim.x * blockDim.x;
    uint64_t head = words;  // differently aligned source and destination: all scalar
    if ((((uintptr_t)s ^ (uintptr_t)d) & 15) == 0) {
        const uint64_t to16 = ((16 - ((uintptr_t)d & 15)) & 15) / 4;
        head = to16 < words ? to16 : words;
    }
    for (uint64_t i = tid; i < head; i += nthr) d[i] = s[i];
    const uint64_t q = (words - head) / 4;
    const uint4* __restrict__ s4 = reinterpret_cast<const uint4*>(s + head);
    uint4* __restrict__ d4 = reinterpret_cast<uint4*>(d + head);
    for (uint64_t i = tid; i < q; i += nthr) __stcs(d4 + i, __ldcs(s4 + i));
    for (uint64_t i = head + q * 4 + tid; i < words; i += nthr) d[i] = s[i];
}
// Two names for one copy, so that a trace tells the delta's hops apart from the other lists': pack_kernel copies the phase A / B
// lists (24 blocks per segment), bulk_copy_kernel the visible delta's, up to hundreds of MB per tick (DESIGN §8, bulk_copy_grid).
__global__ void __launch_bounds__(COPY_THREADS) pack_kernel(PackArgs a) { copy_segment(a); }
__global__ void __launch_bounds__(COPY_THREADS) bulk_copy_kernel(PackArgs a) { copy_segment(a); }
// x blocks per segment: enough for one 16-byte vector per thread, at most `per_sm4` quarters of the SM count; y: the segments.
// Hop 1 (HBM -> HBM) takes 8 (2 CTAs per SM and segment: a launch of the four delta segments holds at most 8 per SM), hop 2 (HBM ->
// PCIe) 1: its CTAs stay resident for the whole transfer (4 ms on the all-entities-move workload); at 8 the pipelined tick took
// 6.03 ms there, at 1 5.5-5.6 ms, at the same PCIe rate (DESIGN §8).
dim3 bulk_copy_grid(const chd_engine* e, const PackArgs& a, uint64_t per_sm4) {
    uint64_t words = 1;
    for (int k = 0; k < a.n; k++) words = std::max<uint64_t>(words, std::max(a.seg[k].cap, a.seg[k].fixed) * a.seg[k].elem_words);
    const uint64_t x = std::min<uint64_t>(blocks_for((words + 3) / 4, COPY_THREADS), per_sm4 * (uint64_t)e->sm_count / 4);
    return dim3((unsigned)std::max<uint64_t>(x, 1), (unsigned)a.n);
}
// What an asynchronous fetch snapshots of the last delta: its list lengths and whether it overflowed (then nothing is copied)
struct DeltaHead {
    unsigned long long n_entered, n_left, overflow;  // (travel to the pinned header in this order)
    unsigned long long copy_entered, copy_left, copy_offsets;
};
constexpr uint32_t DELTA_HEADER_WORD = 32;  // byte 128 of the pinned header
static_assert(sizeof(Counters) <= DELTA_HEADER_WORD * 4 && DELTA_HEADER_WORD * 4 + 24 + 4 <= CHD_FETCH_HEADER_BYTES, "pinned header layout");
__global__ void delta_head_kernel(const unsigned long long* n_entered, const unsigned long long* n_left, uint64_t enter_cap, uint64_t leave_cap,
                                  const uint32_t* bad_ids, uint32_t n_out, DeltaHead* h) {
    const unsigned long long ne = *n_entered, nl = *n_left;
    const bool ovf = chd_delta_overflowed(ne, nl, enter_cap, leave_cap, bad_ids && *bad_ids);
    h->n_entered = ne;
    h->n_left = nl;
    h->overflow = ovf;
    h->copy_entered = ovf ? 0 : ne;
    h->copy_left = ovf ? 0 : nl;
    h->copy_offsets = ovf ? 0 : (unsigned long long)n_out + 1;
}
// The start of a fetch set's staging buffer: the counts hop 2 sizes its copies by, as hop 1 (or delta_head_kernel) saw them
struct StageHead {
    Counters a, b;     // the counters when phase A / phase B is final (b also travels to the pinned header)
    uint32_t n_pairs;  // the pair lists' length, pair_off[n_slots]
    DeltaHead delta;
};
bool is_pinned_host(const void* p) {
    if (!p) return true;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeHost;
}
// deltas enqueued since the previous fetch, which this fetch (with or without delta buffers) now accounts for
uint32_t take_deltas(chd_engine* e, bool want) {
    chd_engine::Delta& D = e->dl;
    const uint64_t k = D.seq - D.fetched;
    D.fetched = D.seq;
    return want ? (uint32_t)std::min<uint64_t>(k, 0xFFFFFFFFu) : 0;
}
// Synchronous form: the last delta's list lengths, read on `s` once it has finished there; *overflow: no lists to copy
chd_status read_delta_counts(chd_engine* e, cudaStream_t s, uint32_t deltas, chd_delta_counts* dc, bool* overflow) {
    const chd_engine::Delta& D = e->dl;
    *dc = chd_delta_counts{};
    *overflow = false;
    if (!deltas) return CHD_OK;
    DeltaLengths dn;
    const chd_status st = chd_read_delta_lengths(e, s, &dn);
    if (st != CHD_OK) return st;
    *dc = chd_delta_counts{dn.n_entered, dn.n_left, D.n_out, deltas};
    *overflow = chd_delta_overflowed(dn.n_entered, dn.n_left, D.enter_cap, D.leave_cap, dn.bad_ids);
    return CHD_OK;
}
// When a tick's results are final, for the read-back streams of both fetches (the synchronous one's early form and the asynchronous
// one).  Phase A: after the interest fill (ev_pairs) and the build: pairs, interest diff, query statuses, handover list, cell CSR.
chd_status wait_phase_a(chd_engine* e, cudaStream_t s) {
    CU(e, cudaStreamWaitEvent(s, e->ev_pairs, 0));
    if (e->build_done_recorded) CU(e, cudaStreamWaitEvent(s, e->ev_build_done, 0));
    return CHD_OK;
}
// Phase B: after the aux chain (ev_join: fan-out) and the emit preparation (ev_prep_done): due list, visible offsets, counters.  And
// after the visible delta, because its CHD_OVF_DELTA belongs to this tick's summary: a tick's delta off the engine stream (ev_done)
// and, when the fetch reads deltas back, the last delta wherever it ran (ev_end; a standalone one runs on the engine stream).
chd_status wait_phase_b(chd_engine* e, cudaStream_t s, bool deltas) {
    CU(e, cudaStreamWaitEvent(s, e->ev_join, 0));
    CU(e, cudaStreamWaitEvent(s, e->ev_prep_done, 0));
    if (e->dl.done_recorded) CU(e, cudaStreamWaitEvent(s, e->dl.ev_done, 0));
    if (deltas) CU(e, cudaStreamWaitEvent(s, e->dl.ev_end, 0));
    return CHD_OK;
}
}  // namespace

extern "C" {

chd_status chd_get_cells(chd_engine* e, uint32_t* cell_start, uint32_t* sorted_entity) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    const uint32_t C = e->g.cells;
    const CopySet& c = chd_copy_in(e);
    if (cell_start) CU(e, cudaMemcpyAsync(cell_start, c.cell_start, sizeof(uint32_t) * ((uint64_t)C + 1), cudaMemcpyDefault, e->stream));
    if (sorted_entity) {
        uint32_t nin = 0;
        chd_status st = chd_read_u32(e, c.cell_start + C, &nin);
        if (st != CHD_OK) return st;
        CU(e, cudaMemcpyAsync(sorted_entity, chd_sorted_out(e, c), sizeof(uint32_t) * nin, cudaMemcpyDefault, e->stream));
    }
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

chd_status chd_get_pairs(chd_engine* e, uint32_t* pair_off, uint32_t* channel_id, uint32_t* dist, uint32_t* interval_ms, uint8_t* flags,
                         int64_t* last_fanout_ns, uint64_t* last_message_index) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    uint32_t P = 0;
    chd_status st = chd_read_u32(e, pb.off + S, &P);
    if (st != CHD_OK) return st;
    if (P > e->lim.max_pairs) return CHD_ERR_CAPACITY;
    cudaStream_t s = e->stream;
    if (pair_off) CU(e, cudaMemcpyAsync(pair_off, pb.off, sizeof(uint32_t) * ((uint64_t)S + 1), cudaMemcpyDefault, s));
    if (channel_id) {
        add_const_kernel<<<blocks_for(P ? P : 1, 256), 256, 0, s>>>(pb.cell, P, e->g.id_start, e->d_vcnt);
        KCHECK(e);
        CU(e, cudaMemcpyAsync(channel_id, e->d_vcnt, sizeof(uint32_t) * P, cudaMemcpyDefault, s));
    }
    if (dist) CU(e, cudaMemcpyAsync(dist, pb.dist, sizeof(uint32_t) * P, cudaMemcpyDefault, s));
    if (interval_ms) CU(e, cudaMemcpyAsync(interval_ms, pb.interval, sizeof(uint32_t) * P, cudaMemcpyDefault, s));
    if (flags) CU(e, cudaMemcpyAsync(flags, pb.flags, P, cudaMemcpyDefault, s));
    if (last_fanout_ns) CU(e, cudaMemcpyAsync(last_fanout_ns, pb.last, sizeof(int64_t) * P, cudaMemcpyDefault, s));
    if (last_message_index) CU(e, cudaMemcpyAsync(last_message_index, pb.last_index, sizeof(uint64_t) * P, cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

chd_status chd_get_query_status(chd_engine* e, uint32_t* status, uint32_t n) {
    if (!e || !status) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    if (n > e->last_nq) n = e->last_nq;
    CU(e, cudaMemcpyAsync(status, e->d_status, sizeof(uint32_t) * n, cudaMemcpyDefault, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

chd_status chd_get_diff(chd_engine* e, uint32_t* new_sub, uint32_t* new_channel, uint32_t* unsub_sub, uint32_t* unsub_channel) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    const uint32_t nn = e->h_ctr->n_sub_new, nu = e->h_ctr->n_unsub;
    cudaStream_t s = e->stream;
    if (new_sub) CU(e, cudaMemcpyAsync(new_sub, e->d_new_sub, sizeof(uint32_t) * nn, cudaMemcpyDefault, s));
    if (new_channel) CU(e, cudaMemcpyAsync(new_channel, e->d_new_ch, sizeof(uint32_t) * nn, cudaMemcpyDefault, s));
    if (unsub_sub) CU(e, cudaMemcpyAsync(unsub_sub, e->d_gone_sub, sizeof(uint32_t) * nu, cudaMemcpyDefault, s));
    if (unsub_channel) CU(e, cudaMemcpyAsync(unsub_channel, e->d_gone_ch, sizeof(uint32_t) * nu, cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

chd_status chd_get_visible(chd_engine* e, uint64_t* vis_off, uint32_t* vis_entity) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    const uint32_t S = e->n_slots;
    cudaStream_t s = e->stream;
    if (vis_off) CU(e, cudaMemcpyAsync(vis_off, e->d_vis_off, sizeof(uint64_t) * ((uint64_t)S + 1), cudaMemcpyDefault, s));
    if (vis_entity) {
        uint64_t* h64 = (uint64_t*)e->h_get;
        CU(e, cudaMemcpyAsync(h64, e->d_vis_off + S, 8, cudaMemcpyDeviceToHost, s));
        CU(e, cudaStreamSynchronize(s));
        const uint64_t V = *h64;
        if (V > e->lim.max_visible) return CHD_ERR_CAPACITY;
        CU(e, cudaMemcpyAsync(vis_entity, e->d_vis, sizeof(uint32_t) * V, cudaMemcpyDefault, s));
    }
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

chd_status chd_get_visible_slot(chd_engine* e, uint32_t slot, uint32_t* out, uint64_t cap, uint64_t* count) {
    if (!e || !count || slot >= e->n_slots) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    uint64_t* h64 = (uint64_t*)e->h_get;
    CU(e, cudaMemcpyAsync(h64, e->d_vis_off + slot, 16, cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    const uint64_t b = h64[0], n = h64[1] - h64[0];
    *count = n;
    if (h64[1] > e->lim.max_visible) return CHD_ERR_CAPACITY;
    const uint64_t m = n < cap ? n : cap;
    if (m && out) {
        CU(e, cudaMemcpyAsync(out, e->d_vis + b, sizeof(uint32_t) * m, cudaMemcpyDefault, e->stream));
        CU(e, cudaStreamSynchronize(e->stream));
    }
    return CHD_OK;
}

chd_status chd_get_due(chd_engine* e, chd_due* out, uint32_t cap) {
    if (!e || !out) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    uint32_t n = e->h_ctr->n_due;
    if (n > e->lim.max_due) n = e->lim.max_due;  // the list overflowed (CHD_OVF_DUE): what fitted + CHD_DUE_VOID holes
    if (n > cap) n = cap;
    CU(e, cudaMemcpyAsync(out, e->d_due, sizeof(chd_due) * n, cudaMemcpyDefault, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

chd_status chd_get_handover(chd_engine* e, uint32_t* entity, uint32_t* src_channel, uint32_t* dst_channel, uint32_t cap) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    uint32_t n = 0;
    chd_status st = chd_read_u32(e, &e->d_ctr->n_handover, &n);
    if (st != CHD_OK) return st;
    if (n > e->ho_cap) n = e->ho_cap;
    if (n > cap) n = cap;
    cudaStream_t s = e->stream;
    if (entity) CU(e, cudaMemcpyAsync(entity, e->d_ho_entity, sizeof(uint32_t) * n, cudaMemcpyDefault, s));
    if (src_channel) CU(e, cudaMemcpyAsync(src_channel, e->d_ho_src, sizeof(uint32_t) * n, cudaMemcpyDefault, s));
    if (dst_channel) CU(e, cudaMemcpyAsync(dst_channel, e->d_ho_dst, sizeof(uint32_t) * n, cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

chd_status chd_fetch_results(chd_engine* e, const chd_result_buffers* b, chd_tick_summary* summary) {
    return chd_fetch_results_delta(e, b, nullptr, summary, nullptr);
}

chd_status chd_fetch_results_delta(chd_engine* e, const chd_result_buffers* b, const chd_delta_buffers* dbuf, chd_tick_summary* summary,
                                   chd_delta_counts* counts) {
    if (!e || !b || !summary) return CHD_ERR_INVALID;
    if (dbuf && !e->dl.on) {
        e->fail("chd_fetch_results_delta: delta buffers before chd_reserve_visible_delta");
        return CHD_ERR_STATE;
    }
    CHD_ENTER(e, ENTRY_DEVICE);
    // only a fetch of the expanded list waits for the copy kernel: the other results are final once the tick's head has run
    if (b->vis_entity) CU(e, chd_copy_wait(e));
    chd_status st;
    cudaStream_t s = e->stream;
    cudaStream_t main_stream = e->stream;
    const bool early = e->early_ready;
    const uint32_t deltas = take_deltas(e, dbuf != nullptr);
    chd_delta_counts dc{};
    bool delta_ovf = false;
    if (counts) *counts = dc;
    // error exits: no copy into the caller's buffers may still be in flight when this returns
    auto drain = [&](chd_status r) {
        cudaStreamSynchronize(e->dl_stream);
        cudaStreamSynchronize(e->dl_stream_b);
        cudaStreamSynchronize(main_stream);
        return r;
    };
    // the delta's counts are known (they are reported on every exit from here on); checks the caller's capacities before any
    // delta buffer is written
    auto delta_check = [&]() -> chd_status {
        if (counts) *counts = dc;
        if (!deltas) return CHD_OK;
        if (delta_ovf) {
            e->fail("chd_fetch_results_delta: the visible delta overflowed (CHD_OVF_DELTA / CHD_OVF_DELTA_IDS): %llu entered / %llu left",
                    (unsigned long long)dc.n_entered, (unsigned long long)dc.n_left);
            return CHD_ERR_CAPACITY;
        }
        if (((dbuf->enter_off || dbuf->leave_off) && dbuf->slot_cap < (uint64_t)dc.n_slots + 1) ||
            (dbuf->enter_entity && dc.n_entered > dbuf->entity_cap) || (dbuf->leave_entity && dc.n_left > dbuf->entity_cap)) {
            e->fail("chd_fetch_results_delta: %u slots, %llu entered / %llu left do not fit slot_cap %llu / entity_cap %llu", dc.n_slots,
                    (unsigned long long)dc.n_entered, (unsigned long long)dc.n_left, (unsigned long long)dbuf->slot_cap,
                    (unsigned long long)dbuf->entity_cap);
            return CHD_ERR_CAPACITY;
        }
        return CHD_OK;
    };
    Counters ca{};  // counters as of phase A
    if (early) {
        // The tick is probably still running.  Read back on separate streams, phase A and then phase B, each as soon as its results
        // are final (wait_phase_a / wait_phase_b), while the emit kernel is still writing the expanded list.
        s = e->dl_stream;
        st = wait_phase_a(e, s);
        if (st != CHD_OK) return st;
        CU(e, cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
        CU(e, cudaStreamSynchronize(s));  // sync A
        ca = *e->h_ctr;
        if (ca.overflow & CHD_OVF_PAIRS) {  // the pair arrays are incomplete: report through the full summary
            CU(e, cudaStreamSynchronize(main_stream));
            st = read_delta_counts(e, main_stream, deltas, &dc, &delta_ovf);
            if (st != CHD_OK) return st;
            if (counts) *counts = dc;
            return chd_summary(e, summary);
        }
    } else {
        st = chd_summary(e, summary);  // sync #1 (also surfaces capacity overflows)
        if (st == CHD_OK || st == CHD_ERR_CAPACITY) {  // (the delta, if any, ran on the engine stream or was joined into it)
            const chd_status r = read_delta_counts(e, s, deltas, &dc, &delta_ovf);
            if (r != CHD_OK) return r;
            const chd_status dchk = delta_check();
            if (st == CHD_OK) st = dchk;
        }
        if (st != CHD_OK) return st;
        ca.n_pairs = summary->n_pairs; ca.n_sub_new = summary->n_sub_new; ca.n_unsub = summary->n_unsub;
        ca.n_handover = summary->n_handover; ca.n_entities_in_world = summary->n_entities_in_world;
    }
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = ca.n_pairs;
    if ((b->pair_channel || b->pair_dist || b->pair_interval_ms) && P > b->pair_cap) {
        e->fail("chd_fetch_results: %llu pairs > pair_cap %llu", (unsigned long long)P, (unsigned long long)b->pair_cap);
        return drain(CHD_ERR_CAPACITY);
    }
    if (b->pair_off) CU(e, cudaMemcpyAsync(b->pair_off, pb.off, sizeof(uint32_t) * ((uint64_t)S + 1), cudaMemcpyDefault, s));
    if (b->pair_channel && e->pair_ch_valid) {
        CU(e, cudaMemcpyAsync(b->pair_channel, e->d_pair_ch, sizeof(uint32_t) * P, cudaMemcpyDefault, s));
    } else if (b->pair_channel) {
        add_const_kernel<<<blocks_for(P ? P : 1, 256), 256, 0, main_stream>>>(pb.cell, (uint32_t)P, e->g.id_start, e->d_vcnt);
        KCHECK(e);
        CU(e, cudaMemcpyAsync(b->pair_channel, e->d_vcnt, sizeof(uint32_t) * P, cudaMemcpyDefault, main_stream));
    }
    if (b->pair_dist) CU(e, cudaMemcpyAsync(b->pair_dist, pb.dist, sizeof(uint32_t) * P, cudaMemcpyDefault, s));
    if (b->pair_interval_ms) CU(e, cudaMemcpyAsync(b->pair_interval_ms, pb.interval, sizeof(uint32_t) * P, cudaMemcpyDefault, s));
    const uint64_t nn = ca.n_sub_new, nu = ca.n_unsub;
    if ((b->new_sub || b->new_channel) && nn > b->diff_cap) return drain(CHD_ERR_CAPACITY);
    if ((b->unsub_sub || b->unsub_channel) && nu > b->diff_cap) return drain(CHD_ERR_CAPACITY);
    if (b->new_sub) CU(e, cudaMemcpyAsync(b->new_sub, e->d_new_sub, sizeof(uint32_t) * nn, cudaMemcpyDefault, s));
    if (b->new_channel) CU(e, cudaMemcpyAsync(b->new_channel, e->d_new_ch, sizeof(uint32_t) * nn, cudaMemcpyDefault, s));
    if (b->unsub_sub) CU(e, cudaMemcpyAsync(b->unsub_sub, e->d_gone_sub, sizeof(uint32_t) * nu, cudaMemcpyDefault, s));
    if (b->unsub_channel) CU(e, cudaMemcpyAsync(b->unsub_channel, e->d_gone_ch, sizeof(uint32_t) * nu, cudaMemcpyDefault, s));
    if (b->handover_entity || b->handover_src || b->handover_dst) {
        uint32_t nh = ca.n_handover;
        if (nh > e->ho_cap) nh = e->ho_cap;
        if (nh > b->handover_cap) return drain(CHD_ERR_CAPACITY);
        if (b->handover_entity) CU(e, cudaMemcpyAsync(b->handover_entity, e->d_ho_entity, sizeof(uint32_t) * nh, cudaMemcpyDefault, s));
        if (b->handover_src) CU(e, cudaMemcpyAsync(b->handover_src, e->d_ho_src, sizeof(uint32_t) * nh, cudaMemcpyDefault, s));
        if (b->handover_dst) CU(e, cudaMemcpyAsync(b->handover_dst, e->d_ho_dst, sizeof(uint32_t) * nh, cudaMemcpyDefault, s));
    }
    if (b->query_status) {
        const uint32_t n = e->last_nq < b->status_cap ? e->last_nq : b->status_cap;
        CU(e, cudaMemcpyAsync(b->query_status, e->d_status, sizeof(uint32_t) * n, cudaMemcpyDefault, s));
    }
    if (b->cell_start) CU(e, cudaMemcpyAsync(b->cell_start, chd_copy_in(e).cell_start, sizeof(uint32_t) * ((uint64_t)e->g.cells + 1), cudaMemcpyDefault, s));
    if (b->sorted_entity) {
        if (ca.n_entities_in_world > b->entity_cap) return drain(CHD_ERR_CAPACITY);
        CU(e, cudaMemcpyAsync(b->sorted_entity, chd_sorted_out(e, chd_copy_in(e)), sizeof(uint32_t) * (uint64_t)ca.n_entities_in_world, cudaMemcpyDefault, s));
    }
    cudaStream_t sa = s;  // stream carrying the phase-A copies
    if (early) {  // phase B, on its own stream: its counter read-back must not queue behind the phase-A copies
        s = e->dl_stream_b;
        st = wait_phase_b(e, s, deltas);
        if (st != CHD_OK) return st;
        CU(e, cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
        CU(e, cudaStreamSynchronize(s));  // sync B
        st = chd_decode_summary(e, summary);
        if (st == CHD_OK || st == CHD_ERR_CAPACITY) {
            const chd_status r = read_delta_counts(e, s, deltas, &dc, &delta_ovf);
            if (r != CHD_OK) return drain(r);
            const chd_status dchk = delta_check();
            if (st == CHD_OK) st = dchk;
        }
        if (st != CHD_OK) return drain(st);
    }
    if (deltas) {  // the delta is final on `s`; its counts were checked against the caller's capacities
        const chd_engine::Delta& D = e->dl;
        const uint64_t off_bytes = 8ull * ((uint64_t)dc.n_slots + 1);
        if (dbuf->enter_off) CU(e, cudaMemcpyAsync(dbuf->enter_off, D.enter_off, off_bytes, cudaMemcpyDefault, s));
        if (dbuf->leave_off) CU(e, cudaMemcpyAsync(dbuf->leave_off, D.leave_off, off_bytes, cudaMemcpyDefault, s));
        if (dbuf->enter_entity && dc.n_entered) CU(e, cudaMemcpyAsync(dbuf->enter_entity, D.enter, 4ull * dc.n_entered, cudaMemcpyDefault, s));
        if (dbuf->leave_entity && dc.n_left) CU(e, cudaMemcpyAsync(dbuf->leave_entity, D.leave, 4ull * dc.n_left, cudaMemcpyDefault, s));
    }
    if (b->due) {
        if (summary->n_due > b->due_cap) return drain(CHD_ERR_CAPACITY);
        CU(e, cudaMemcpyAsync(b->due, e->d_due, sizeof(chd_due) * (uint64_t)summary->n_due, cudaMemcpyDefault, s));
    }
    if (b->vis_off) CU(e, cudaMemcpyAsync(b->vis_off, e->d_vis_off, sizeof(uint64_t) * ((uint64_t)S + 1), cudaMemcpyDefault, s));
    if (b->vis_entity) {
        if (summary->n_visible > b->vis_cap) return drain(CHD_ERR_CAPACITY);
        CU(e, cudaMemcpyAsync(b->vis_entity, e->d_vis, sizeof(uint32_t) * summary->n_visible, cudaMemcpyDefault, main_stream));
    }
    CU(e, cudaStreamSynchronize(s));  // last sync of the read-back stream(s)
    if (sa != s) CU(e, cudaStreamSynchronize(sa));
    if (s != main_stream) CU(e, cudaStreamSynchronize(main_stream));  // the tick itself (expanded list) has finished
    return CHD_OK;
}

chd_status chd_fetch_results_async(chd_engine* e, const chd_result_buffers* b, void* pinned_header) {
    return chd_fetch_results_async_delta(e, b, nullptr, pinned_header);
}

chd_status chd_fetch_results_async_delta(chd_engine* e, const chd_result_buffers* b, const chd_delta_buffers* dbuf, void* pinned_header) {
    if (!e || !b || !pinned_header) return CHD_ERR_INVALID;
    if (!e->early_ready) {
        e->fail("chd_fetch_results_async needs a two-stream tick (chd_tick with emit, or chd_begin_interest + chd_tick) just before it");
        return CHD_ERR_STATE;
    }
    if (b->vis_entity) {
        e->fail("chd_fetch_results_async does not copy the expanded list (use chd_fetch_results / chd_get_visible)");
        return CHD_ERR_INVALID;
    }
    if (dbuf && !e->dl.on) {
        e->fail("chd_fetch_results_async_delta: delta buffers before chd_reserve_visible_delta");
        return CHD_ERR_STATE;
    }
    const chd_delta_buffers nod{};
    const chd_delta_buffers& db = dbuf ? *dbuf : nod;
    for (const void* p : {(const void*)b->pair_off, (const void*)b->pair_channel, (const void*)b->pair_dist, (const void*)b->pair_interval_ms, (const void*)b->new_sub,
                          (const void*)b->new_channel, (const void*)b->unsub_sub, (const void*)b->unsub_channel, (const void*)b->due, (const void*)b->handover_entity,
                          (const void*)b->handover_src, (const void*)b->handover_dst, (const void*)b->query_status, (const void*)b->vis_off,
                          (const void*)b->cell_start, (const void*)b->sorted_entity, (const void*)pinned_header, (const void*)db.enter_off,
                          (const void*)db.leave_off, (const void*)db.enter_entity, (const void*)db.leave_entity})
        if (!is_pinned_host(p)) {
            e->fail("chd_fetch_results_async: every buffer must be pinned host memory (chd_alloc_pinned)");
            return CHD_ERR_INVALID;
        }
    CHD_ENTER(e, ENTRY_DEVICE);
    if (e->fetch_issued - e->fetch_waited >= 2) {
        e->fail("chd_fetch_results_async: two fetches are already outstanding (call chd_fetch_wait)");
        return CHD_ERR_STATE;
    }
    const int fi = (int)(e->fetch_issued & 1);
    chd_engine::Delta& D = e->dl;
    const uint32_t deltas = take_deltas(e, dbuf != nullptr);
    if (!e->ev_fetch_a[fi] && !(chd_make_event(e, &e->ev_fetch_a[fi]) && chd_make_event(e, &e->ev_fetch_b[fi]))) return CHD_ERR_CUDA;
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    Counters* ctr = e->d_ctr;
    uint32_t* hdr = reinterpret_cast<uint32_t*>(pinned_header);
    uint32_t* truncated = hdr + CHD_FETCH_HEADER_BYTES / 4 - 1;
    *truncated = 0;  // (host write, ordered before the kernels are launched)
    memset(hdr + DELTA_HEADER_WORD, 0, 24);  // the delta's counts (stay 0 when this fetch carries none)
    // ---- hop 1: snapshot into device staging (microseconds: the next tick is ordered after THIS, not after the PCIe transfer);
    //      hop 2: staging -> the caller's pinned buffers on a stream of its own, sized by the snapshot's own copy of the counts.
    // Each list is declared once, and its staging slice, hop-1 segment and hop-2 segment all come from that declaration.  Staging
    // addresses are byte offsets until the buffer has been sized.
    enum { HOP_A, HOP_B, HOP_DELTA };  // the hop-1 launch that snapshots a list: phase A, phase B, the visible delta
    struct Count {
        const void* live;  // what hop 1 reads (nullptr: the snapshot's, which delta_head_kernel writes before hop 1; or `fixed`)
        int64_t snap;      // what hop 2 reads: offset in StageHead (-1: `fixed`)
        uint32_t is64;
        uint64_t fixed;
    };
    struct List {
        int hop;
        const void* src;  // nullptr: no hop 1 (delta_head_kernel writes the slice)
        void* dst;        // nullptr: no hop 2 (a count only hop 2 reads)
        Count n;
        uint64_t cap;
        uint32_t words;   // element size in 32-bit words
        uint64_t slice;   // offset in the staging buffer
    };
    List lists[24];
    int nl = 0;
    auto up16 = [](uint64_t v) { return (v + 15) & ~(uint64_t)15; };
    uint64_t stage_bytes = up16(sizeof(StageHead));
    auto list = [&](int hop, const void* src, void* dst, Count n, uint64_t cap, uint32_t words) {  // a requested list: a slice of its own
        if (!dst) return;
        lists[nl++] = List{hop, src, dst, n, cap, words, stage_bytes};
        stage_bytes += up16(std::max(cap, n.fixed) * words * 4);
    };
    auto count = [&](int hop, const void* src, void* dst, uint64_t at, uint32_t words) {  // a count: its slice is its place in StageHead
        lists[nl++] = List{hop, src, dst, Count{nullptr, -1, 0, words}, words, 1, at};
    };
    auto fixed = [](uint64_t n) { return Count{nullptr, -1, 0, n}; };
#define SNAP(field) (int64_t)offsetof(StageHead, field)
    const uint64_t S1 = (uint64_t)S + 1, C1 = (uint64_t)e->g.cells + 1, hcap = std::min<uint64_t>(b->handover_cap, e->ho_cap);
    // list(hop, device source, pinned destination, count: live and in the snapshot, capacity, element words)
    list(HOP_A, pb.off, b->pair_off, fixed(S1), S1, 1);
    list(HOP_A, e->d_pair_ch, b->pair_channel, {pb.off + S, SNAP(n_pairs)}, b->pair_cap, 1);
    list(HOP_A, pb.dist, b->pair_dist, {pb.off + S, SNAP(n_pairs)}, b->pair_cap, 1);
    list(HOP_A, pb.interval, b->pair_interval_ms, {pb.off + S, SNAP(n_pairs)}, b->pair_cap, 1);
    list(HOP_A, e->d_new_sub, b->new_sub, {&ctr->n_sub_new, SNAP(a.n_sub_new)}, b->diff_cap, 1);
    list(HOP_A, e->d_new_ch, b->new_channel, {&ctr->n_sub_new, SNAP(a.n_sub_new)}, b->diff_cap, 1);
    list(HOP_A, e->d_gone_sub, b->unsub_sub, {&ctr->n_unsub, SNAP(a.n_unsub)}, b->diff_cap, 1);
    list(HOP_A, e->d_gone_ch, b->unsub_channel, {&ctr->n_unsub, SNAP(a.n_unsub)}, b->diff_cap, 1);
    list(HOP_A, e->d_status, b->query_status, fixed(std::min<uint64_t>(e->last_nq, b->status_cap)), b->status_cap, 1);
    list(HOP_A, chd_copy_in(e).cell_start, b->cell_start, fixed(C1), C1, 1);
    list(HOP_A, chd_sorted_out(e, chd_copy_in(e)), b->sorted_entity, {&ctr->n_entities_in_world, SNAP(a.n_entities_in_world)}, b->entity_cap, 1);
    list(HOP_A, e->d_ho_entity, b->handover_entity, {&ctr->n_handover, SNAP(a.n_handover)}, hcap, 1);
    list(HOP_A, e->d_ho_src, b->handover_src, {&ctr->n_handover, SNAP(a.n_handover)}, hcap, 1);
    list(HOP_A, e->d_ho_dst, b->handover_dst, {&ctr->n_handover, SNAP(a.n_handover)}, hcap, 1);
    list(HOP_B, e->d_due, b->due, {&ctr->n_due, SNAP(b.n_due)}, std::min<uint64_t>(b->due_cap, e->lim.max_due), sizeof(chd_due) / 4);
    list(HOP_B, e->d_vis_off, b->vis_off, fixed(S1), S1, 2);
    count(HOP_A, ctr, nullptr, SNAP(a), sizeof(Counters) / 4);
    count(HOP_A, pb.off + S, nullptr, SNAP(n_pairs), 1);
    count(HOP_B, ctr, pinned_header, SNAP(b), sizeof(Counters) / 4);
    if (deltas) {  // the lengths each delta copy moves are 0 after an overflow
        list(HOP_DELTA, D.enter_off, db.enter_off, {nullptr, SNAP(delta.copy_offsets), 1}, db.slot_cap, 2);
        list(HOP_DELTA, D.leave_off, db.leave_off, {nullptr, SNAP(delta.copy_offsets), 1}, db.slot_cap, 2);
        list(HOP_DELTA, D.enter, db.enter_entity, {nullptr, SNAP(delta.copy_entered), 1}, db.entity_cap, 1);
        list(HOP_DELTA, D.leave, db.leave_entity, {nullptr, SNAP(delta.copy_left), 1}, db.entity_cap, 1);
        count(HOP_DELTA, nullptr, hdr + DELTA_HEADER_WORD, SNAP(delta), 6);  // its lengths and overflow
        if (!e->dl_stream_d && !chd_make_stream(e, &e->dl_stream_d)) return CHD_ERR_CUDA;
    }
#undef SNAP
    if (!ensure_cap(e, &e->d_fetch_stage[fi], &e->fetch_stage_bytes[fi], stage_bytes, stage_bytes)) return CHD_ERR_CUDA;
    if (!e->dl_stream_c && !chd_make_stream(e, &e->dl_stream_c)) return CHD_ERR_CUDA;
    if (!e->ev_fetch_done[fi] && !chd_make_event(e, &e->ev_fetch_done[fi])) return CHD_ERR_CUDA;
    uint8_t* const stage = e->d_fetch_stage[fi];
    PackArgs hop1[3] = {}, hop2[3] = {};
    for (int k = 0; k < nl; k++) {
        const List& l = lists[k];
        void* slice = stage + l.slice;
        const void* snap = l.n.snap < 0 ? nullptr : stage + l.n.snap;
        PackArgs &h1 = hop1[l.hop], &h2 = hop2[l.hop];
        if (l.src) h1.seg[h1.n++] = PackSeg{l.src, slice, l.n.live ? l.n.live : snap, l.n.fixed, l.cap, l.words, l.n.is64};
        if (l.dst) h2.seg[h2.n++] = PackSeg{slice, l.dst, snap, l.n.fixed, l.cap, l.words, l.n.is64};
    }
    for (int h = 0; h < 3; h++) hop1[h].truncated = hop2[h].truncated = truncated;
    cudaStream_t sa = e->dl_stream, sb = e->dl_stream_b, sc = e->dl_stream_c;
    chd_status st = wait_phase_a(e, sa);
    if (st != CHD_OK) return st;
    pack_kernel<<<dim3(24, (unsigned)hop1[HOP_A].n), COPY_THREADS, 0, sa>>>(hop1[HOP_A]);
    KCHECK(e);
    CU(e, cudaEventRecord(e->ev_fetch_a[fi], sa));
    CU(e, cudaStreamWaitEvent(sc, e->ev_fetch_a[fi], 0));
    const bool prof = e->profiling == 1;
    if (prof) CU(e, cudaEventRecord(e->evt(CHD_STAGE_READBACK, e->stage_n[CHD_STAGE_READBACK], 0), sc));
    if (hop2[HOP_A].n) {
        pack_kernel<<<dim3(24, (unsigned)hop2[HOP_A].n), COPY_THREADS, 0, sc>>>(hop2[HOP_A]);
        KCHECK(e);
    }
    st = wait_phase_b(e, sb, deltas);
    if (st != CHD_OK) return st;
    if (deltas) {
        // hop 1 of the delta on a stream of its own, from the delta's end on: beside the expanded-list kernel, and only the next delta
        // waits for it (D.read_guard), not the next tick's other stages
        const cudaStream_t sd = e->dl_stream_d;
        CU(e, cudaStreamWaitEvent(sd, D.ev_end, 0));
        delta_head_kernel<<<1, 1, 0, sd>>>(reinterpret_cast<const unsigned long long*>(D.enter_off + D.n_out),
                                          reinterpret_cast<const unsigned long long*>(D.leave_off + D.n_out), D.enter_cap, D.leave_cap,
                                          D.ids ? D.bad_ids : nullptr, D.n_out, &reinterpret_cast<StageHead*>(stage)->delta);
        KCHECK(e);
        if (hop1[HOP_DELTA].n) {
            bulk_copy_kernel<<<bulk_copy_grid(e, hop1[HOP_DELTA], 8), COPY_THREADS, 0, sd>>>(hop1[HOP_DELTA]);
            KCHECK(e);
        }
        CU(e, cudaEventRecord(D.ev_read[fi], sd));
        D.read_guard = true;
        D.read_fi = fi;
    }
    pack_kernel<<<dim3(24, (unsigned)hop1[HOP_B].n), COPY_THREADS, 0, sb>>>(hop1[HOP_B]);
    KCHECK(e);
    CU(e, cudaEventRecord(e->ev_fetch_b[fi], sb));
    CU(e, cudaStreamWaitEvent(sc, e->ev_fetch_b[fi], 0));
    pack_kernel<<<dim3(24, (unsigned)hop2[HOP_B].n), COPY_THREADS, 0, sc>>>(hop2[HOP_B]);
    KCHECK(e);
    if (deltas) {
        CU(e, cudaStreamWaitEvent(sc, D.ev_read[fi], 0));
        bulk_copy_kernel<<<bulk_copy_grid(e, hop2[HOP_DELTA], 1), COPY_THREADS, 0, sc>>>(hop2[HOP_DELTA]);
        KCHECK(e);
    }
    CU(e, cudaEventRecord(e->ev_fetch_done[fi], sc));
    if (prof) {
        CU(e, cudaEventRecord(e->evt(CHD_STAGE_READBACK, e->stage_n[CHD_STAGE_READBACK], 1), sc));
        e->stage_n[CHD_STAGE_READBACK]++;
    }
    e->fetch_guard = true;  // the next tick's kernels are ordered after these copies (they overwrite the arrays being read)
    e->fetch_header[fi] = pinned_header;
    e->fetch_deltas[fi] = deltas;
    e->fetch_delta_slots[fi] = deltas ? D.n_out : 0;
    e->fetch_issued++;
    return CHD_OK;
}

chd_status chd_fetch_wait(chd_engine* e, chd_tick_summary* summary) { return chd_fetch_wait_delta(e, summary, nullptr); }

chd_status chd_fetch_wait_delta(chd_engine* e, chd_tick_summary* summary, chd_delta_counts* counts) {
    if (!e || !summary) return CHD_ERR_INVALID;
    if (e->fetch_issued == e->fetch_waited) {
        e->fail("chd_fetch_wait without a chd_fetch_results_async in flight");
        return CHD_ERR_STATE;
    }
    CHD_ENTER(e, ENTRY_DEVICE);
    const int fi = (int)(e->fetch_waited & 1);  // the OLDEST outstanding fetch
    CU(e, cudaEventSynchronize(e->ev_fetch_done[fi]));
    e->fetch_waited++;
    static_assert(sizeof(Counters) + 4 <= CHD_FETCH_HEADER_BYTES, "CHD_FETCH_HEADER_BYTES too small");
    memcpy(e->h_ctr, e->fetch_header[fi], sizeof(Counters));
    const uint32_t truncated = reinterpret_cast<const uint32_t*>(e->fetch_header[fi])[CHD_FETCH_HEADER_BYTES / 4 - 1];
    chd_status st = chd_decode_summary(e, summary);
    const unsigned long long* dh = reinterpret_cast<const unsigned long long*>(reinterpret_cast<const uint32_t*>(e->fetch_header[fi]) + DELTA_HEADER_WORD);
    const uint32_t deltas = e->fetch_deltas[fi];
    if (counts) *counts = deltas ? chd_delta_counts{dh[0], dh[1], e->fetch_delta_slots[fi], deltas} : chd_delta_counts{};
    if (st == CHD_OK && deltas && dh[2]) {
        e->fail("chd_fetch_results_async_delta: the visible delta overflowed (CHD_OVF_DELTA / CHD_OVF_DELTA_IDS): %llu entered / %llu left",
                dh[0], dh[1]);
        return CHD_ERR_CAPACITY;
    }
    if (st == CHD_OK && truncated) {
        e->fail("chd_fetch_results_async: a result list did not fit its buffer (truncated)");
        return CHD_ERR_CAPACITY;
    }
    return st;
}

chd_status chd_device_view(chd_engine* e, int which, void** d_ptr, uint64_t* count) {
    if (!e || !d_ptr) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);  // work the caller orders after this on the engine stream sees the final arrays
    PairBuf& pb = e->pairs[e->cur];
    uint64_t c = 0;
    void* p = nullptr;
    switch (which) {
        case CHD_VIEW_CELL_START: p = chd_copy_in(e).cell_start; c = (uint64_t)e->g.cells + 2; break;
        case CHD_VIEW_SORTED_ENTITY: p = (void*)chd_sorted_out(e, chd_copy_in(e)); c = e->n_sorted; break;
        case CHD_VIEW_ENT_CELL: p = e->d_key; c = e->n_own + e->n_halo; break;
        case CHD_VIEW_PAIR_OFF: p = pb.off; c = (uint64_t)e->n_slots + 1; break;
        case CHD_VIEW_PAIR_CHANNEL: p = pb.cell; c = e->lim.max_pairs; break;
        case CHD_VIEW_PAIR_DIST: p = pb.dist; c = e->lim.max_pairs; break;
        case CHD_VIEW_VIS_OFF: p = e->d_vis_off; c = (uint64_t)e->n_slots + 1; break;
        case CHD_VIEW_VIS_ENTITY: p = e->d_vis; c = e->lim.max_visible; break;
        case CHD_VIEW_DUE: p = e->d_due; c = e->lim.max_due; break;
        case CHD_VIEW_DELTA_ENTER_OFF: p = e->dl.enter_off; c = (uint64_t)e->dl.n_out + 1; break;
        case CHD_VIEW_DELTA_ENTER: p = e->dl.enter; c = e->dl.enter_cap; break;
        case CHD_VIEW_DELTA_LEAVE_OFF: p = e->dl.leave_off; c = (uint64_t)e->dl.n_out + 1; break;
        case CHD_VIEW_DELTA_LEAVE: p = e->dl.leave; c = e->dl.leave_cap; break;
        case CHD_VIEW_ENTITY_ID: p = e->tbl.d_id_of_slot; c = e->tbl.hw; break;
        default: return CHD_ERR_INVALID;
    }
    if (which == CHD_VIEW_ENTITY_ID && !e->tbl.on) {
        e->fail("chd_device_view: CHD_VIEW_ENTITY_ID needs entity-table mode (chd_entity_table_init)");
        return CHD_ERR_STATE;
    }
    if (which >= CHD_VIEW_DELTA_ENTER_OFF && which <= CHD_VIEW_DELTA_LEAVE && !e->dl.on) {
        e->fail("chd_device_view: no visible delta before chd_reserve_visible_delta");
        return CHD_ERR_STATE;
    }
    *d_ptr = p;
    if (count) *count = c;
    return CHD_OK;
}
}  // extern "C"
