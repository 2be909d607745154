// chd_tick.cu — expanded visible lists, fan-out, and Channel.Tick for every spatial channel as one batched, two-stream tick.
#include "chd_engine.h"

#include "chd_emit.cuh"
#include "chd_fanout.cuh"
#include "chd_misc.cuh"

extern "C" {

// Which copy kernel (host-known inputs only: nothing here waits for the device):
//   CTA tiles + per-tile descriptors  when cells are large against a tile (<= 2 segments per tile is the common case)
//                                     AND the world holds at most L2 / 32 entities (1.6 M with the H100's 50 MB): the size
//                                     bound separates config #2 (1 M entities, CTA tiles) from config #3 (10 M, warp tiles)
//                                     and has not been re-tuned for the 4-byte-per-entity sources;
//   warp tiles (round 1's kernel)     otherwise: many segments per tile (config #5) or a world above that bound (config #3).
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
    const int set = e->pf_copy.cur;
    const CopySet& c = chd_copy_in(e);
    const uint64_t key = stage_key(0x656d6974ull, S, e->cur, cta_tiles, s, set);
    // the preparation rewrites its copy-input set: after the last copy kernel that read it (a tick without a build reuses the set
    // of the copy before it; after a build this is the copy the build already waited for)
    chd_status st = chd_pf_after_read(e, e->pf_copy, set, s);
    if (st == CHD_OK) st = chd_epoch_tick(e, s, EP_EMIT);
    // the tiles the partition may describe: tile_desc / general_tiles hold one entry per CTA tile of max_visible (+ 8), first_pair
    // one per warp tile, so a visible count far above max_visible (CHD_OVF_VISIBLE) never writes past either
    const uint64_t tile_cap = cta_tiles ? (e->lim.max_visible + EMIT_TILE - 1) / EMIT_TILE + 1 : e->max_tiles;
    if (st != CHD_OK) return st;
    return run_stage(e, s, e->g_emit_prep, key, [&]() -> chd_status {
        // per-pair visible counts are computed by the scan itself; the partition pass opens the next epoch
        SCAN(e, exclusive_scan_fn<PairVcountIn, uint64_t>(PairVcountIn{pb.cell, c.cell_start}, c.voff, P, e->site_voff, s, pb.off + S));
        emit_partition_kernel<<<grid, 256, 0, s>>>(pb.off + S, P, c.voff, pb.cell, c.cell_start, c.first_pair, cta_tiles ? c.tile_desc : nullptr,
                                                   tile_cap, S, pb.off, e->d_vis_off, e->lim.max_visible, e->d_ctr, e->d_epoch + EP_EMIT, tile,
                                                   c.general_tiles, c.n_general, c.n_visible);
        KCHECK(e);
        return CHD_OK;
    });
}

// the copy kernels on `s`; they read V from their set, which the next tick's preparation does not rewrite while they run
static chd_status emit_kernel_enqueue(chd_engine* e, cudaStream_t s, bool cta_tiles) {
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = e->lim.max_pairs;
    const int set = e->pf_copy.cur;
    const CopySet& c = chd_copy_in(e);
    chd_status st = chd_pf_wait(e, e->pf_copy, s);
    if (st != CHD_OK) return st;
    {
    StageTimer kt(e, s, CHD_STAGE_EMIT_KERNEL);
    if (cta_tiles) {
        // EMIT_TILES_PER_CTA tiles per CTA, dispatched by the hardware block scheduler.  The tile count lives on the device; the grid is
        // sized from the last visible count the host has seen (+3 %: the kernel loops if that was too few, surplus CTAs exit
        // at once), from the capacity before that.
        const uint64_t cap_tiles = (e->lim.max_visible + EMIT_TILE - 1) / EMIT_TILE;
        uint64_t tiles = e->vis_estimate ? std::min<uint64_t>(cap_tiles, (e->vis_estimate + e->vis_estimate / 32) / EMIT_TILE + 64) : cap_tiles;
        if (tiles == 0) tiles = 1;
        if (tiles > 0x7fffffffull) tiles = 0x7fffffffull;
        tiles = (tiles + EMIT_TILES_PER_CTA - 1) / EMIT_TILES_PER_CTA;
        emit_visible_kernel<<<(unsigned)tiles, EMIT_THREADS, CHD_EMIT_DYN_SMEM, s>>>(c.n_visible, chd_sorted_out(e, c), c.tile_desc, e->d_vis, e->lim.max_visible);
        KCHECK(e);
        emit_visible_general_kernel<<<(unsigned)e->sm_count * 2, EMIT_THREADS, 0, s>>>(c.general_tiles, c.n_general, pb.off + S, P, c.n_visible,
                                                                                       c.voff, pb.cell, c.cell_start, chd_sorted_out(e, c),
                                                                                       c.first_pair, e->d_vis, e->lim.max_visible);
    } else {
        emit_visible_warp_kernel<<<(unsigned)e->sm_count * 4, EMIT_THREADS, 0, s>>>(pb.off + S, P, c.voff, pb.cell, c.cell_start, chd_sorted_out(e, c),
                                                                                    c.first_pair, e->d_vis, e->lim.max_visible);
    }
    KCHECK(e);
    }
    st = chd_pf_note_read(e, e->pf_copy, set, s);
    if (st != CHD_OK) return st;
    e->copy_pending = s == e->stream ? -1 : set;
    return CHD_OK;
}

// The emit: the preparation (ending with ev_prep_done), then the copy kernel on `s`, after `kernel_ev` if one is given.  Without
// `pairs_ev` the preparation runs on `s` too.  In a two-stream tick it needs only the new pairs (`pairs_ev`, second stream) and
// the cell CSR OFFSETS (ev_counts: recorded between the two halves of a single-pass build), not the sorted entity array — it runs
// on prep_stream next to the build's scatter; the copy kernel follows on `s` (copy_stream) when both and the build
// (ev_build_done) are done.
static chd_status emit_enqueue(chd_engine* e, cudaStream_t s, cudaEvent_t pairs_ev, cudaEvent_t kernel_ev) {
    if (!e->built) {
        e->fail("emit before any chd_build");
        return CHD_ERR_STATE;
    }
    const bool cta_tiles = emit_uses_cta_tiles(e);
    StageTimer timer(e, s, CHD_STAGE_EMIT);
    const cudaStream_t ps = pairs_ev ? e->prep_stream : s;
    if (pairs_ev) {
        CU(e, cudaStreamWaitEvent(ps, e->ev_counts, 0));
        CU(e, cudaStreamWaitEvent(ps, pairs_ev, 0));
    }
    chd_status st = emit_prep_enqueue(e, ps, cta_tiles);
    if (st != CHD_OK) return st;
    CU(e, cudaEventRecord(e->ev_prep_done, ps));  // visible offsets + counters are final; only the expanded list is still to come
    if (pairs_ev) {
        CU(e, cudaStreamWaitEvent(s, e->ev_prep_done, 0));
        CU(e, cudaStreamWaitEvent(s, e->ev_build_done, 0));
    }
    if (kernel_ev) CU(e, cudaStreamWaitEvent(s, kernel_ev, 0));
    return emit_kernel_enqueue(e, s, cta_tiles);
}

chd_status chd_emit_visible(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD);
    return emit_enqueue(e, e->stream, nullptr, nullptr);
}

chd_status chd_set_channel_start_times(chd_engine* e, const int64_t* start_ns) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_no_chain(e, "chd_set_channel_start_times", false) != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    if (!start_ns) {
        e->have_cell_start = false;
        return CHD_OK;
    }
    CU(e, cudaMemcpyAsync(e->d_cell_start_ns, start_ns, sizeof(int64_t) * (uint64_t)e->g.cells, cudaMemcpyDefault, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    e->have_cell_start = true;
    return CHD_OK;
}

static chd_status fanout_enqueue(chd_engine* e, cudaStream_t s, int64_t t_ns) {
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = e->lim.max_pairs;
    StageTimer timer(e, s, CHD_STAGE_FANOUT);
    chd_status st = chd_pf_wait(e, e->rings.pf, s);  // rings handed over by chd_adopt_prefetched: ordered after their upload
    if (st == CHD_OK) st = chd_ring_total_flush(e, s);
    if (st != CHD_OK) return st;
    chd_epoch_tick(e, s, EP_FANOUT);
    e->rings.after_fanout = false;
    stage_begin_kernel<<<1, 1, 0, s>>>(e->d_time + 1, t_ns, e->d_epoch + EP_FANOUT, &e->d_ctr->n_due, 1, nullptr);
    KCHECK(e);
    const RingDev ring = chd_ring_view(e);
    const unsigned grid = (unsigned)e->sm_count * 16;
    // the graph bakes in the slot count, the pair-buffer parity and the ring pointers
    const uint64_t key = stage_key(0x66616eull, S, e->cur, ring.channel_msg_index != nullptr, ring.off, ring.end, ring.arrival, ring.sender, ring.index,
                                   ring.channel_msg_index, ring.start);
    st = run_stage(e, s, e->g_fanout, key, [&]() -> chd_status {
        const unsigned blocks = (unsigned)std::min<uint64_t>((P + 127) / 128, (uint64_t)e->sm_count * 16);
        fanout_kernel<<<blocks ? blocks : 1, 128, 0, s>>>(pb.off + S, P, pb, e->d_conn, ring, e->d_time + 1, e->g.id_start, e->d_by_cell, e->d_due,
                                                          e->d_due_key, e->lim.max_due, e->d_ctr);
        KCHECK(e);
        return CHD_OK;
    });
    return st != CHD_OK ? st : chd_pf_note_read(e, e->rings.pf, e->rings.pf.cur, s);
}

chd_status chd_fanout_tick(chd_engine* e, int64_t t_ns) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD);
    return fanout_enqueue(e, e->stream, t_ns);
}

chd_status chd_adopt_prefetched(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    if (e->pf_pos.staged < 0 && e->pf_q.staged < 0 && e->rings.pf.staged < 0) {
        e->fail("chd_adopt_prefetched without a preceding chd_prefetch_entities / chd_prefetch_queries / chd_prefetch_rings");
        return CHD_ERR_STATE;
    }
    if (e->pf_q.staged >= 0 && chd_rule_no_generated_batch(e, "chd_adopt_prefetched of a query batch") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    chd_pf_adopt(e->pf_q);  // consumed by the next chd_begin_interest / chd_update_interest called with q == NULL
    chd_rings_adopt(e);
    if (!chd_pf_adopt(e->pf_pos)) return CHD_OK;
    chd_status st = chd_pf_wait(e, e->pf_pos, e->stream);
    if (st != CHD_OK) return st;
    e->in_place = {};
    chd_entities_replaced(e, chd_pos_front(e).n);
    return CHD_OK;
}

chd_status chd_summary(chd_engine* e, chd_tick_summary* out) {
    if (!e || !out) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(Counters), cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return chd_decode_summary(e, out);
}

chd_status chd_decode_summary(chd_engine* e, chd_tick_summary* out) {
    const Counters& c = *e->h_ctr;
    if (e->tbl.on) chd_table_observe(e, c.delta_build);
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
    if (!q && chd_rule_batch_waiting(e, "chd_begin_interest", false) != CHD_OK) return CHD_ERR_STATE;
    if (chd_rule_no_chain(e, "chd_begin_interest", false) != CHD_OK || chd_rule_rings_staged(e, "chd_begin_interest") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_FETCH_GUARD);
    const chd_status st = aux_chain_enqueue(e, e->stream, q, true, t_ns, with_fanout != 0);
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

// Dependency graph of a tick:   build ----------------+--> emit preparation --> copy kernel
//                               interest --> fan-out  |      (the emit needs the cell CSR and the new pairs)
// The build runs on build_stream, the interest / fan-out chain on aux_stream (started here or earlier by chd_begin_interest),
// the emit preparation on prep_stream: the tick's head, all forked from the engine stream `s` (= e->stream) at high priority.
// The copy kernel (HBM-bound) runs on copy_stream at the lowest priority.  `s` joins everything but the copy kernel, and the
// previous tick's copy kernel: the next tick's head runs beside this tick's copy, and `s` is never more than one copy behind
// (chd_copy_wait joins the rest).  A tick with nothing to overlap runs its stages one after the other on `s`.
static chd_status tick_enqueue(chd_engine* e, cudaStream_t s, const chd_query_batch* q, int64_t t_ns, uint32_t flags) {
    chd_status st;
    const bool need_build = (flags & CHD_TICK_BUILD) && (e->entities_dirty || !e->built);
    const bool do_emit = flags & CHD_TICK_EMIT;
    const bool do_fanout = flags & CHD_TICK_FANOUT;
    const bool do_delta = flags & CHD_TICK_VISIBLE_DELTA;
    const bool started = e->interest_pending;  // the aux chain of this tick was started by chd_begin_interest
    const bool follow = flags & CHD_TICK_FOLLOW;  // the batch is the generated one (q == NULL)
    if (follow && q) return CHD_ERR_INVALID;
    if (follow && !started && chd_rule_batch_waiting(e, "chd_tick", true) != CHD_OK) return CHD_ERR_STATE;
    const bool interest = q || follow;  // this tick has an interest update of its own
    e->early_ready = false;
    e->build_done_recorded = false;
    e->dl.done_recorded = false;
    if (started && interest) {
        e->fail("chd_tick: a query batch was given while chd_begin_interest is pending");
        return CHD_ERR_STATE;
    }
    if (do_delta && chd_delta_check(e, need_build) != CHD_OK) return CHD_ERR_STATE;
    if (!started && !((interest || do_fanout) && (need_build || do_emit))) {
        CU(e, chd_copy_wait(e));  // one stream: the whole tick runs after the previous tick's copy kernel
        if (need_build) {
            st = chd_build_on(e, s);
            if (st != CHD_OK) return st;
        }
        if (interest) {
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
        return do_delta ? chd_delta_on(e, s) : CHD_OK;
    }
    if (!started) {
        st = aux_chain_enqueue(e, s, q, interest, t_ns, do_fanout);
        if (st != CHD_OK) return st;
    }
    const bool fanout_done = started ? e->pending_fanout : do_fanout;
    e->interest_pending = false;
    // the build forks off `s` onto build_stream: left on `s`, it would queue behind the previous copy kernel's grid
    const cudaStream_t bs = e->build_stream;
    CU(e, cudaEventRecord(e->ev_fork, s));
    CU(e, cudaStreamWaitEvent(bs, e->ev_fork, 0));
    CU(e, chd_copy_wait(e));  // `s` (not the head, forked above) waits for the previous tick's copy kernel
    if (need_build) {
        st = chd_build_on(e, bs);
        if (st != CHD_OK) return st;
        e->build_done_recorded = true;
    }
    CU(e, cudaEventRecord(e->ev_build_done, bs));
    if (do_delta) CU(e, cudaEventRecord(e->dl.ev_in, bs));  // the cell CSR and keys of this tick (or of the last build) are final
    if (do_emit) {
        // the preparation waits for the new pairs (for the fork when this tick updates no interest); CHD_TICK_EARLY_RESULTS: the
        // copy kernel starts after the whole aux chain, so every host-facing result is final while it is still streaming
        st = emit_enqueue(e, e->copy_stream, (started || interest) ? e->ev_pairs : e->ev_interest,
                          (flags & CHD_TICK_EARLY_RESULTS) ? e->ev_join : nullptr);
        if (st != CHD_OK) return st;
        CU(e, cudaStreamWaitEvent(s, e->ev_prep_done, 0));
    }
    if (do_delta) {
        // latency-bound: on prep_stream (after the emit preparation), next to the expanded-list kernel and the aux chain; it needs
        // the build and the new pairs, and the engine stream waits for it
        const cudaStream_t ds = e->prep_stream;
        CU(e, cudaStreamWaitEvent(ds, e->dl.ev_in, 0));
        if (started || interest) CU(e, cudaStreamWaitEvent(ds, e->ev_pairs, 0));
        st = chd_delta_on(e, ds);
        if (st != CHD_OK) return st;
        CU(e, cudaEventRecord(e->dl.ev_done, ds));
        e->dl.done_recorded = true;  // the early read-back's counters wait for it (CHD_OVF_DELTA belongs to this tick's summary)
        CU(e, cudaStreamWaitEvent(s, e->dl.ev_done, 0));
    }
    CU(e, cudaStreamWaitEvent(s, e->ev_build_done, 0));
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
    if (chd_rule_rings_staged(e, "chd_tick") != CHD_OK) return CHD_ERR_STATE;
    chd_status st;
    {
        // from the tick's first head kernel to the end of its copy kernel (without the summary read-back)
        StageTimer whole(e, e->stream, CHD_STAGE_TICK);
        CHD_ENTER(e, ENTRY_FETCH_GUARD);
        st = tick_enqueue(e, e->stream, q, t_ns, flags);
        if (e->copy_pending >= 0) whole.s = e->copy_stream;
    }
    if (st != CHD_OK) return st;
    if (out) return chd_summary(e, out);
    return CHD_OK;
}
}  // extern "C"
