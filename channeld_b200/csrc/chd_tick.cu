// chd_tick.cu — expanded visible lists, update rings, fan-out, and Channel.Tick for every spatial channel as one batched,
// two-stream tick.
#include "chd_engine.h"

#include "chd_emit.cuh"
#include "chd_fanout.cuh"
#include "chd_misc.cuh"
#include "chd_rings.cuh"

extern "C" {

// Which copy kernel (host-known inputs only: nothing here waits for the device):
//   CTA tiles + per-tile descriptors  when cells are large against a tile (<= 2 segments per tile is the common case)
//                                     AND the CSR's four phase copies fit in half the L2 (they stay resident next to the write
//                                     stream: the copy is then a pure write stream);
//   warp tiles (round 1's kernel)     otherwise: many segments per tile (config #5) or sources streamed from DRAM (config #3).
static bool emit_uses_cta_tiles(const chd_engine* e) {
    const uint64_t n_build = (uint64_t)e->n_own + (e->halo_on_device ? (uint64_t)e->border_cap : (uint64_t)e->n_halo);
    const uint64_t own_cells = (uint64_t)(e->g.col_hi - e->g.col_lo) * e->g.rows;  // (the whole grid on one GPU, the slab on N)
    return (uint64_t)e->n_own / (own_cells ? own_cells : 1) >= (uint64_t)EMIT_TILE / 2 && n_build * 16ull <= (uint64_t)e->l2_bytes / 2;
}

// emit preparation on `s`: per-pair output offsets (scan), per-tile first pairs / descriptors, per-subscriber offsets, V
static chd_status emit_prep_enqueue(chd_engine* e, cudaStream_t s, bool cta_tiles) {
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = e->lim.max_pairs;
    const unsigned grid = (unsigned)e->sm_count * 8;
    const uint32_t tile = cta_tiles ? (uint32_t)EMIT_TILE : (uint32_t)EMIT_WARP_TILE;
    const uint64_t key = mix_key(mix_key(mix_key(mix_key(0x656d6974ull, S), (uint64_t)e->cur), cta_tiles), (uint64_t)(uintptr_t)s);
    chd_status st = chd_epoch_tick(e, s, EP_EMIT);
    if (st != CHD_OK) return st;
    return run_stage(e, s, e->g_emit_prep[e->cur], key, [&]() -> chd_status {
        // per-pair visible counts are computed by the scan itself; the partition pass opens the next epoch
        SCAN(e, exclusive_scan_fn<PairVcountIn, uint64_t>(PairVcountIn{pb.cell, e->d_cell_start}, e->d_voff, P, e->site_voff, s, pb.off + S));
        emit_partition_kernel<<<grid, 256, 0, s>>>(pb.off + S, P, e->d_voff, pb.cell, e->d_cell_start, e->d_first_pair, cta_tiles ? e->d_tile_desc : nullptr,
                                                   e->max_tiles, S, pb.off, e->d_vis_off, e->lim.max_visible, e->d_ctr, e->d_epoch + EP_EMIT, tile,
                                                   e->d_general_tiles, e->d_n_general);
        KCHECK(e);
        return CHD_OK;
    });
}

static chd_status emit_kernel_enqueue(chd_engine* e, cudaStream_t s, bool cta_tiles) {
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = e->lim.max_pairs;
    StageTimer kt(e, s, CHD_STAGE_EMIT_KERNEL);
    if (cta_tiles) {
        // One CTA per tile, dispatched by the hardware block scheduler.  The tile count lives on the device; the grid is
        // sized from the last visible count the host has seen (+3 %: the kernel loops if that was too few, surplus CTAs exit
        // at once), from the capacity before that.
        const uint64_t cap_tiles = (e->lim.max_visible + EMIT_TILE - 1) / EMIT_TILE;
        uint64_t tiles = e->vis_estimate ? std::min<uint64_t>(cap_tiles, (e->vis_estimate + e->vis_estimate / 32) / EMIT_TILE + 64) : cap_tiles;
        if (tiles == 0) tiles = 1;
        if (tiles > 0x7fffffffull) tiles = 0x7fffffffull;
        tiles = (tiles + EMIT_TILES_PER_CTA - 1) / EMIT_TILES_PER_CTA;
        emit_visible_kernel<<<(unsigned)tiles, EMIT_THREADS, CHD_EMIT_DYN_SMEM, s>>>(&e->d_ctr->n_visible, e->d_sorted4, e->d_tile_desc, e->d_vis, e->lim.max_visible);
        KCHECK(e);
        emit_visible_general_kernel<<<(unsigned)e->sm_count * 2, EMIT_THREADS, 0, s>>>(e->d_general_tiles, e->d_n_general, pb.off + S, P, &e->d_ctr->n_visible,
                                                                                       e->d_voff, pb.cell, e->d_cell_start, e->d_sorted4, e->phase_stride,
                                                                                       e->d_first_pair, e->d_vis, e->lim.max_visible);
    } else {
        emit_visible_warp_kernel<<<(unsigned)e->sm_count * 4, EMIT_THREADS, 0, s>>>(pb.off + S, P, e->d_voff, pb.cell, e->d_cell_start, e->d_sorted4,
                                                                                    e->phase_stride, e->d_first_pair, e->d_vis, e->lim.max_visible);
    }
    KCHECK(e);
    return CHD_OK;
}

// The emit: the preparation (ending with ev_prep_done), then the copy kernel on `s`, after `kernel_ev` if one is given.  Without
// `pairs_ev` the preparation runs on `s` too.  In a two-stream tick it needs only the new pairs (`pairs_ev`, second stream) and
// the cell CSR OFFSETS (ev_counts: recorded between the two halves of a single-pass build), not the sorted entity array — it runs
// on prep_stream next to the build's scatter; the copy kernel follows on `s` when both are done.
static chd_status emit_enqueue(chd_engine* e, cudaStream_t s, cudaEvent_t pairs_ev, cudaEvent_t kernel_ev) {
    if (!e->built) {
        e->fail("emit before any chd_build");
        return CHD_ERR_STATE;
    }
    const bool cta_tiles = emit_uses_cta_tiles(e);
    StageTimer timer(e, s, CHD_STAGE_EMIT);
    const cudaStream_t ps = pairs_ev ? e->prep_stream : s;
    if (pairs_ev) {
        CU(e, cudaStreamWaitEvent(ps, e->ev_fork, 0));    // the previous tick's copy kernel (it reads what the preparation rewrites)
        CU(e, cudaStreamWaitEvent(ps, e->ev_counts, 0));
        CU(e, cudaStreamWaitEvent(ps, pairs_ev, 0));
    }
    chd_status st = emit_prep_enqueue(e, ps, cta_tiles);
    if (st != CHD_OK) return st;
    CU(e, cudaEventRecord(e->ev_prep_done, ps));  // visible offsets + counters are final; only the expanded list is still to come
    if (pairs_ev) CU(e, cudaStreamWaitEvent(s, e->ev_prep_done, 0));
    if (kernel_ev) CU(e, cudaStreamWaitEvent(s, kernel_ev, 0));
    return emit_kernel_enqueue(e, s, cta_tiles);
}

chd_status chd_emit_visible(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    CU(e, cudaSetDevice(e->device));
    chd_status st = chd_fetch_guard(e, e->stream);
    return st != CHD_OK ? st : emit_enqueue(e, e->stream, nullptr, nullptr);
}

chd_status chd_set_rings(chd_engine* e, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival, const uint32_t* sender,
                         const uint64_t* index, const uint64_t* ch_msg_index) {
    if (!e || !ring_off) return CHD_ERR_INVALID;
    if (e->rings_owned) {
        e->fail("chd_set_rings: the rings are device-owned (chd_rings_init): use chd_rings_append");
        return CHD_ERR_STATE;
    }
    CU(e, cudaSetDevice(e->device));
    const uint32_t C = e->g.cells;
    const uint32_t total = n_entries;
    if (total > e->lim.max_ring_entries) {
        e->fail("%u ring entries > max_ring_entries %u", total, e->lim.max_ring_entries);
        return CHD_ERR_CAPACITY;
    }
    if (total && (!arrival || !sender || !index)) return CHD_ERR_INVALID;
    const bool in_place = chd_is_device_ptr(e, ring_off) && (!total || (chd_is_device_ptr(e, arrival) && chd_is_device_ptr(e, sender) && chd_is_device_ptr(e, index))) &&
                          (!ch_msg_index || chd_is_device_ptr(e, ch_msg_index));
    if (in_place) {  // device-resident rings: consumed in place
        e->ring_off_p = ring_off; e->ring_arrival_p = arrival; e->ring_sender_p = sender; e->ring_index_p = index;
        e->ch_msg_index_p = ch_msg_index;
    } else {
        CU(e, cudaMemcpyAsync(e->d_ring_off, ring_off, sizeof(uint32_t) * ((uint64_t)C + 1), cudaMemcpyDefault, e->stream));
        if (total) {
            CU(e, cudaMemcpyAsync(e->d_ring_arrival, arrival, sizeof(int64_t) * total, cudaMemcpyDefault, e->stream));
            CU(e, cudaMemcpyAsync(e->d_ring_sender, sender, sizeof(uint32_t) * total, cudaMemcpyDefault, e->stream));
            CU(e, cudaMemcpyAsync(e->d_ring_index, index, sizeof(uint64_t) * total, cudaMemcpyDefault, e->stream));
        }
        if (ch_msg_index) CU(e, cudaMemcpyAsync(e->d_ch_msg_index, ch_msg_index, sizeof(uint64_t) * C, cudaMemcpyDefault, e->stream));
        e->ring_off_p = e->d_ring_off; e->ring_arrival_p = e->d_ring_arrival; e->ring_sender_p = e->d_ring_sender;
        e->ring_index_p = e->d_ring_index; e->ch_msg_index_p = ch_msg_index ? e->d_ch_msg_index : nullptr;
    }
    e->have_ch_msg_index = ch_msg_index != nullptr;
    e->ring_set = -1;
    e->wait_rings = false;
    // the fan-out kernel clamps ring_off to this: a lying caller cannot cause out-of-bounds reads
    set_u32_kernel<<<1, 1, 0, e->stream>>>(e->d_ring_total, total);
    KCHECK(e);
    return CHD_OK;
}

/* ---- device-owned rings: ChannelData.OnUpdate's buffer maintenance on the GPU (data.go:149-173) */

chd_status chd_rings_init(chd_engine* e, uint32_t capacity_per_cell) {
    if (!e || capacity_per_cell <= RING_MAX_BUFFER) {
        if (e) e->fail("chd_rings_init: capacity_per_cell must exceed %u (MaxUpdateMsgBufferSize: the reference's buffer may grow beyond it)", RING_MAX_BUFFER);
        return CHD_ERR_INVALID;
    }
    const uint64_t need = (uint64_t)e->g.cells * capacity_per_cell;
    if (need > e->lim.max_ring_entries) {
        e->fail("chd_rings_init: %u cells x %u entries > max_ring_entries %u", e->g.cells, capacity_per_cell, e->lim.max_ring_entries);
        return CHD_ERR_CAPACITY;
    }
    CU(e, cudaSetDevice(e->device));
    cudaStream_t s = e->stream;
    rings_init_kernel<<<blocks_for((uint64_t)e->g.cells + 1, 128), 128, 0, s>>>(e->g.cells, capacity_per_cell, e->d_rb_begin, e->d_rb_end);
    KCHECK(e);
    CU(e, cudaMemsetAsync(e->d_ch_msg_index, 0, (uint64_t)e->g.cells * 8, s));
    set_u32_kernel<<<1, 1, 0, s>>>(e->d_ring_total, (uint32_t)need);
    KCHECK(e);
    e->rings_owned = true;
    e->ring_cap = capacity_per_cell;
    e->have_ch_msg_index = true;
    e->ring_set = -1;
    e->wait_rings = false;
    return CHD_OK;
}

chd_status chd_rings_append(chd_engine* e, const uint32_t* upd_off, uint32_t n_updates, const int64_t* arrival_ns, const uint32_t* sender_conn_id) {
    if (!e || !upd_off || (n_updates && (!arrival_ns || !sender_conn_id))) return CHD_ERR_INVALID;
    if (!e->rings_owned) {
        e->fail("chd_rings_append before chd_rings_init");
        return CHD_ERR_STATE;
    }
    CU(e, cudaSetDevice(e->device));
    cudaStream_t s = e->stream;
    const uint32_t C = e->g.cells;
    const uint64_t grown = (uint64_t)n_updates + n_updates / 2 + 1024;
    if (!ensure_cap(e, &e->d_upd_arrival, &e->upd_arrival_cap, n_updates, grown) || !ensure_cap(e, &e->d_upd_sender, &e->upd_sender_cap, n_updates, grown))
        return CHD_ERR_CUDA;
    CU(e, cudaMemcpyAsync(e->d_upd_off, upd_off, sizeof(uint32_t) * ((uint64_t)C + 1), cudaMemcpyDefault, s));
    if (n_updates) {
        CU(e, cudaMemcpyAsync(e->d_upd_arrival, arrival_ns, sizeof(int64_t) * n_updates, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(e->d_upd_sender, sender_conn_id, sizeof(uint32_t) * n_updates, cudaMemcpyDefault, s));
    }
    rings_append_kernel<<<blocks_for(C, 128), 128, 0, s>>>(C, e->ring_cap, e->d_upd_off, e->d_upd_arrival, e->d_upd_sender, e->d_rb_begin, e->d_rb_end,
                                                           e->d_ring_arrival, e->d_ring_sender, e->d_ring_index, e->d_ch_msg_index, e->d_cell_max_interval,
                                                           &e->d_ctr->overflow);
    KCHECK(e);
    return CHD_OK;
}

chd_status chd_get_rings(chd_engine* e, uint32_t* ring_off, int64_t* arrival_ns, uint32_t* sender_conn_id, uint64_t* message_index,
                         uint64_t* channel_msg_index, uint32_t cap_entries) {
    if (!e || !ring_off) return CHD_ERR_INVALID;
    if (!e->rings_owned) {
        e->fail("chd_get_rings: the rings are host-owned (chd_set_rings)");
        return CHD_ERR_STATE;
    }
    CU(e, cudaSetDevice(e->device));
    cudaStream_t s = e->stream;
    const uint32_t C = e->g.cells;
    // (control-plane call: a plain two-pass scan through scratch that is free between ticks)
    if (!e->d_ring_scan_scratch && !dalloc(e, &e->d_ring_scan_scratch, scan_scratch_elems(C + 1))) return CHD_ERR_CUDA;
    ring_len_kernel<<<blocks_for(C, 128), 128, 0, s>>>(C, e->d_rb_begin, e->d_rb_end, e->d_upd_off);
    KCHECK(e);
    SCAN(e, exclusive_scan<uint32_t, uint32_t>(e->d_upd_off, e->d_ring_flat_off, C, e->d_ring_scan_scratch, s));
    uint32_t total = 0;
    chd_status st = chd_read_u32(e, e->d_ring_flat_off + C, &total);
    if (st != CHD_OK) return st;
    CU(e, cudaMemcpyAsync(ring_off, e->d_ring_flat_off, sizeof(uint32_t) * ((uint64_t)C + 1), cudaMemcpyDefault, s));
    if (channel_msg_index) CU(e, cudaMemcpyAsync(channel_msg_index, e->d_ch_msg_index, sizeof(uint64_t) * C, cudaMemcpyDefault, s));
    if (arrival_ns || sender_conn_id || message_index) {
        if (total > cap_entries) {
            e->fail("chd_get_rings: %u entries > cap_entries %u", total, cap_entries);
            return CHD_ERR_CAPACITY;
        }
        int64_t* ta = nullptr;
        uint32_t* ts = nullptr;
        uint64_t* ti = nullptr;
        CU(e, cudaMallocAsync((void**)&ta, 8ull * (total + 1), s));
        CU(e, cudaMallocAsync((void**)&ts, 4ull * (total + 1), s));
        CU(e, cudaMallocAsync((void**)&ti, 8ull * (total + 1), s));
        rings_gather_kernel<<<C, 128, 0, s>>>(C, e->d_rb_begin, e->d_rb_end, e->d_ring_flat_off, e->d_ring_arrival, e->d_ring_sender, e->d_ring_index, ta, ts,
                                              ti, total);
        KCHECK(e);
        if (arrival_ns) CU(e, cudaMemcpyAsync(arrival_ns, ta, 8ull * total, cudaMemcpyDefault, s));
        if (sender_conn_id) CU(e, cudaMemcpyAsync(sender_conn_id, ts, 4ull * total, cudaMemcpyDefault, s));
        if (message_index) CU(e, cudaMemcpyAsync(message_index, ti, 8ull * total, cudaMemcpyDefault, s));
        CU(e, cudaFreeAsync(ta, s));
        CU(e, cudaFreeAsync(ts, s));
        CU(e, cudaFreeAsync(ti, s));
    }
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

chd_status chd_set_channel_start_times(chd_engine* e, const int64_t* start_ns) {
    if (!e) return CHD_ERR_INVALID;
    CU(e, cudaSetDevice(e->device));
    if (!start_ns) {
        e->have_cell_start = false;
        return CHD_OK;
    }
    CU(e, cudaMemcpyAsync(e->d_cell_start_ns, start_ns, sizeof(int64_t) * (uint64_t)e->g.cells, cudaMemcpyDefault, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    e->have_cell_start = true;
    return CHD_OK;
}

RingDev chd_ring_view(const chd_engine* e) {
    const int64_t* start = e->have_cell_start ? e->d_cell_start_ns : nullptr;
    if (e->rings_owned)
        return RingDev{e->d_rb_begin, e->d_rb_end, e->d_ring_arrival, e->d_ring_sender, e->d_ring_index, e->d_ch_msg_index, e->d_ring_total, start};
    const uint32_t* off = e->ring_off_p ? e->ring_off_p : e->d_ring_off;
    return RingDev{off, off + 1, e->ring_arrival_p ? e->ring_arrival_p : e->d_ring_arrival, e->ring_sender_p ? e->ring_sender_p : e->d_ring_sender,
                   e->ring_index_p ? e->ring_index_p : e->d_ring_index, e->have_ch_msg_index ? e->ch_msg_index_p : nullptr, e->d_ring_total, start};
}

static chd_status fanout_enqueue(chd_engine* e, cudaStream_t s, int64_t t_ns) {
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = e->lim.max_pairs;
    StageTimer timer(e, s, CHD_STAGE_FANOUT);
    if (e->wait_rings) {  // rings handed over by chd_adopt_prefetched: ordered after their upload
        CU(e, cudaStreamWaitEvent(s, e->ev_upload_rings, 0));
        e->wait_rings = false;
    }
    chd_epoch_tick(e, s, EP_FANOUT);
    stage_begin_kernel<<<1, 1, 0, s>>>(e->d_time + 1, t_ns, e->d_epoch + EP_FANOUT, &e->d_ctr->n_due, 1, nullptr);
    KCHECK(e);
    const RingDev ring = chd_ring_view(e);
    const unsigned grid = (unsigned)e->sm_count * 16;
    uint64_t key = mix_key(mix_key(mix_key(0x66616eull, S), (uint64_t)e->cur), e->have_ch_msg_index);
    for (const void* p : {(const void*)ring.off, (const void*)ring.end, (const void*)ring.arrival, (const void*)ring.sender, (const void*)ring.index,
                          (const void*)ring.channel_msg_index, (const void*)ring.start})
        key = mix_key(key, (uint64_t)(uintptr_t)p);  // pointers are baked into the captured launch
    chd_status st = run_stage(e, s, e->g_fanout[e->cur + (e->ring_set == 1 ? 2 : 0)], key, [&]() -> chd_status {
        const unsigned blocks = (unsigned)std::min<uint64_t>((P + 127) / 128, (uint64_t)e->sm_count * 16);
        fanout_kernel<<<blocks ? blocks : 1, 128, 0, s>>>(pb.off + S, P, pb, e->d_conn, ring, e->d_time + 1, e->g.id_start, e->d_by_cell, e->d_due,
                                                          e->d_due_key, e->lim.max_due, e->d_ctr);
        KCHECK(e);
        return CHD_OK;
    });
    if (st == CHD_OK && e->ring_set >= 0) {
        CU(e, cudaEventRecord(e->ev_ring_read[e->ring_set], s));
        e->ring_read_recorded[e->ring_set] = true;
    }
    return st;
}

chd_status chd_fanout_tick(chd_engine* e, int64_t t_ns) {
    if (!e) return CHD_ERR_INVALID;
    CU(e, cudaSetDevice(e->device));
    chd_status st = chd_fetch_guard(e, e->stream);
    return st != CHD_OK ? st : fanout_enqueue(e, e->stream, t_ns);
}

chd_status chd_prefetch_rings(chd_engine* e, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival, const uint32_t* sender,
                              const uint64_t* index, const uint64_t* ch_msg_index) {
    if (!e || !ring_off) return CHD_ERR_INVALID;
    if (n_entries > e->lim.max_ring_entries) {
        e->fail("%u ring entries > max_ring_entries %u", n_entries, e->lim.max_ring_entries);
        return CHD_ERR_CAPACITY;
    }
    if (n_entries && (!arrival || !sender || !index)) return CHD_ERR_INVALID;
    CU(e, cudaSetDevice(e->device));
    chd_status st = chd_ensure_upload_stream(e);
    if (st != CHD_OK) return st;
    const int set = e->ring_next;
    chd_engine::RStage& r = e->ring_pf[set];
    const uint64_t C = e->g.cells;
    if (!e->ring_pf_alloc[set]) {
        const uint64_t R = e->lim.max_ring_entries;
        if (!(dalloc(e, &r.off, C + 1) && dalloc(e, &r.arrival, R) && dalloc(e, &r.sender, R) && dalloc(e, &r.index, R) && dalloc(e, &r.cmi, C)))
            return CHD_ERR_CUDA;
        e->ring_pf_alloc[set] = true;
    }
    if (e->ring_read_recorded[set]) CU(e, cudaStreamWaitEvent(e->up_stream, e->ev_ring_read[set], 0));
    cudaStream_t us = e->up_stream;
    CU(e, cudaMemcpyAsync(r.off, ring_off, sizeof(uint32_t) * (C + 1), cudaMemcpyDefault, us));
    if (n_entries) {
        CU(e, cudaMemcpyAsync(r.arrival, arrival, sizeof(int64_t) * n_entries, cudaMemcpyDefault, us));
        CU(e, cudaMemcpyAsync(r.sender, sender, sizeof(uint32_t) * n_entries, cudaMemcpyDefault, us));
        CU(e, cudaMemcpyAsync(r.index, index, sizeof(uint64_t) * n_entries, cudaMemcpyDefault, us));
    }
    if (ch_msg_index) CU(e, cudaMemcpyAsync(r.cmi, ch_msg_index, sizeof(uint64_t) * C, cudaMemcpyDefault, us));
    CU(e, cudaEventRecord(e->ev_upload_rings, us));
    e->staged_rings = true;
    e->staged_ring_set = set;
    e->staged_ring_total = n_entries;
    e->staged_ring_cmi = ch_msg_index != nullptr;
    e->ring_next = set ^ 1;
    return CHD_OK;
}

chd_status chd_adopt_prefetched(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    if (!e->staged && !e->staged_q && !e->staged_rings) {
        e->fail("chd_adopt_prefetched without a preceding chd_prefetch_entities / chd_prefetch_queries / chd_prefetch_rings");
        return CHD_ERR_STATE;
    }
    CU(e, cudaSetDevice(e->device));
    if (e->staged_q) {  // consumed by the next chd_begin_interest / chd_update_interest called with q == NULL
        e->adopted_qd = e->staged_qd;
        e->adopted_q_set = e->staged_q_set;
        e->have_adopted_q = true;
        e->wait_q = true;
        e->staged_q = false;
    }
    if (e->staged_rings) {
        const chd_engine::RStage& r = e->ring_pf[e->staged_ring_set];
        e->ring_off_p = r.off; e->ring_arrival_p = r.arrival; e->ring_sender_p = r.sender; e->ring_index_p = r.index;
        e->ch_msg_index_p = e->staged_ring_cmi ? r.cmi : nullptr;
        e->have_ch_msg_index = e->staged_ring_cmi;
        e->ring_set = e->staged_ring_set;
        e->wait_rings = true;
        e->staged_rings = false;
        set_u32_kernel<<<1, 1, 0, e->stream>>>(e->d_ring_total, e->staged_ring_total);
        KCHECK(e);
    }
    if (!e->staged) return CHD_OK;
    CU(e, cudaStreamWaitEvent(e->stream, e->ev_upload, 0));
    e->pos_buf ^= 1;
    e->d_x = e->d_xb[e->pos_buf];
    e->d_z = e->d_zb[e->pos_buf];
    e->pos_x = e->d_x;
    e->pos_z = e->d_z;
    if (e->staged_n != e->n_own) e->have_prev_key = false;
    e->n_own = e->staged_n;
    e->n_halo = 0;
    e->halo_on_device = false;
    e->assigned = false;
    e->entities_dirty = true;
    e->staged = false;
    return CHD_OK;
}

chd_status chd_summary(chd_engine* e, chd_tick_summary* out) {
    if (!e || !out) return CHD_ERR_INVALID;
    CU(e, cudaSetDevice(e->device));
    CU(e, cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return chd_decode_summary(e, out);
}

chd_status chd_decode_summary(chd_engine* e, chd_tick_summary* out) {
    const Counters& c = *e->h_ctr;
    out->n_pairs = c.n_pairs; out->n_visible = c.n_visible; out->n_entities_in_world = c.n_entities_in_world;
    out->n_query_errors = c.n_query_errors; out->n_sub_new = c.n_sub_new; out->n_unsub = c.n_unsub; out->n_kept = c.n_kept;
    out->n_due = c.n_due; out->n_handover = c.n_handover; out->overflow = c.overflow; out->required_pairs = c.required_pairs;
    out->required_window_cells = c.required_window_cells; out->required_visible = c.required_visible; out->required_due = c.n_due;
    out->reserved = 0;
    e->vis_estimate = c.n_visible;  // sizes the next emit grid
    if (c.overflow) {
        e->fail("capacity overflow mask 0x%x (pairs %llu, window cells %llu, visible %llu, due %u required)", c.overflow,
                (unsigned long long)c.required_pairs, (unsigned long long)c.required_window_cells,
                (unsigned long long)c.required_visible, c.n_due);
        // sticky bits are cleared for the next tick; what each overflow leaves behind is specified in chd_gpu.h (CHD_OVF_*)
        CU(e, cudaMemsetAsync(&e->d_ctr->overflow, 0, 4, e->stream));
        return CHD_ERR_CAPACITY;
    }
    return CHD_OK;
}

// Forks the interest / fan-out chain off `s` onto aux_stream: the interest update (if `interest`; q == NULL = the adopted batch),
// ev_interest, the fan-out pass (if `fanout`), ev_join.
static chd_status aux_chain_enqueue(chd_engine* e, cudaStream_t s, const chd_query_batch* q, bool interest, int64_t t_ns, bool fanout) {
    const cudaStream_t aux = e->aux_stream;
    CU(e, cudaEventRecord(e->ev_fork, s));
    CU(e, cudaStreamWaitEvent(aux, e->ev_fork, 0));
    chd_status st = interest ? chd_update_interest_on(e, aux, q, t_ns) : CHD_OK;
    if (st != CHD_OK) return st;
    CU(e, cudaEventRecord(e->ev_interest, aux));
    if (fanout) {
        st = fanout_enqueue(e, aux, t_ns);
        if (st != CHD_OK) return st;
    }
    CU(e, cudaEventRecord(e->ev_join, aux));
    return CHD_OK;
}

chd_status chd_begin_interest(chd_engine* e, const chd_query_batch* q, int64_t t_ns, int with_fanout) {
    if (!e) return CHD_ERR_INVALID;
    if (!q && !e->have_adopted_q) {
        e->fail("chd_begin_interest: q == NULL needs chd_prefetch_queries + chd_adopt_prefetched first");
        return CHD_ERR_STATE;
    }
    if (e->interest_pending) {
        e->fail("chd_begin_interest: the previous one has not been joined by chd_tick yet");
        return CHD_ERR_STATE;
    }
    CU(e, cudaSetDevice(e->device));
    chd_status st = chd_fetch_guard(e, e->stream);
    if (st == CHD_OK) st = aux_chain_enqueue(e, e->stream, q, true, t_ns, with_fanout != 0);
    if (st != CHD_OK) return st;
    e->interest_pending = true;
    e->pending_fanout = with_fanout != 0;
    return CHD_OK;
}

// An asynchronous read-back of the previous tick may still be copying out of the arrays this tick rewrites: order this tick's
// work after it (device-side wait on `s`; in steady state the copies finished long before).
chd_status chd_fetch_guard(chd_engine* e, cudaStream_t s) {
    if (!e->fetch_guard) return CHD_OK;
    const int fi = (int)((e->fetch_issued - 1) & 1);  // the latest fetch (an older one completed before it: same streams)
    CU(e, cudaStreamWaitEvent(s, e->ev_fetch_a[fi], 0));
    CU(e, cudaStreamWaitEvent(s, e->ev_fetch_b[fi], 0));
    e->fetch_guard = false;
    return CHD_OK;
}

// Dependency graph of a tick:   build ----------------+--> emit
//                               interest --> fan-out  |      (emit needs the cell CSR and the new pairs)
// The build / emit chain (HBM-bound) runs on the main stream `s`, the interest / fan-out chain (latency-bound, disjoint state)
// on aux_stream, started here or earlier by chd_begin_interest; the streams are joined before the summary.  A tick with nothing
// to overlap runs its stages one after the other on `s`.
static chd_status tick_enqueue(chd_engine* e, cudaStream_t s, const chd_query_batch* q, int64_t t_ns, uint32_t flags) {
    CU(e, cudaSetDevice(e->device));
    chd_status st = chd_fetch_guard(e, s);
    if (st != CHD_OK) return st;
    const bool need_build = (flags & CHD_TICK_BUILD) && (e->entities_dirty || !e->built);
    const bool do_emit = flags & CHD_TICK_EMIT;
    const bool do_fanout = flags & CHD_TICK_FANOUT;
    const bool started = e->interest_pending;  // the aux chain of this tick was started by chd_begin_interest
    e->early_ready = false;
    e->build_done_recorded = false;
    if (started && q) {
        e->fail("chd_tick: a query batch was given while chd_begin_interest is pending");
        return CHD_ERR_STATE;
    }
    if (!started && !((q || do_fanout) && (need_build || do_emit))) {
        if (need_build) {
            st = chd_build_on(e, s);
            if (st != CHD_OK) return st;
        }
        if (q) {
            st = chd_update_interest_on(e, s, q, t_ns);
            if (st != CHD_OK) return st;
        }
        if (do_emit) {
            st = emit_enqueue(e, s, nullptr, nullptr);
            if (st != CHD_OK) return st;
        }
        if (do_fanout) {
            st = fanout_enqueue(e, s, t_ns);
            if (st != CHD_OK) return st;
        }
        return CHD_OK;
    }
    if (!started) {
        st = aux_chain_enqueue(e, s, q, q != nullptr, t_ns, do_fanout);
        if (st != CHD_OK) return st;
    }
    const bool fanout_done = started ? e->pending_fanout : do_fanout;
    e->interest_pending = false;
    if (need_build) {
        st = chd_build_on(e, s);
        if (st != CHD_OK) return st;
        CU(e, cudaEventRecord(e->ev_build_done, s));
        e->build_done_recorded = true;
    }
    if (do_emit) {
        // the preparation waits for the new pairs (for the fork when this tick updates no interest); CHD_TICK_EARLY_RESULTS: the
        // copy kernel starts after the whole aux chain, so every host-facing result is final while it is still streaming
        st = emit_enqueue(e, s, (started || q) ? e->ev_pairs : e->ev_interest, (flags & CHD_TICK_EARLY_RESULTS) ? e->ev_join : nullptr);
        if (st != CHD_OK) return st;
    }
    CU(e, cudaStreamWaitEvent(s, e->ev_join, 0));
    if (do_fanout && !fanout_done) {
        st = fanout_enqueue(e, s, t_ns);
        if (st != CHD_OK) return st;
    } else {
        e->early_ready = do_emit;  // everything but the expanded list is final at ev_join + ev_prep_done
    }
    return CHD_OK;
}

chd_status chd_tick(chd_engine* e, const chd_query_batch* q, int64_t t_ns, uint32_t flags, chd_tick_summary* out) {
    if (!e) return CHD_ERR_INVALID;
    chd_status st;
    {
        StageTimer whole(e, e->stream, CHD_STAGE_TICK);  // main-stream span of the tick (without the summary read-back)
        st = tick_enqueue(e, e->stream, q, t_ns, flags);
    }
    if (st != CHD_OK) return st;
    if (out) return chd_summary(e, out);
    return CHD_OK;
}
}  // extern "C"
