// chd_delta.cu — visible-set deltas: entered / left entities per subscriber slot since the last successful delta (chd_delta.cuh).
#include "chd_engine.h"

#include "chd_delta.cuh"

static DeltaDev delta_view(chd_engine* e) {
    chd_engine::Delta& D = e->dl;
    const PairBuf& pb = e->pairs[e->cur];
    const CopySet& c = chd_copy_in(e);
    DeltaDev d{};
    d.cells = e->g.cells;
    d.key = e->d_key;
    d.n = e->n_sorted;
    d.cell_start = c.cell_start;
    d.sorted = c.sorted_ent;
    d.pair_off = pb.off;
    d.pair_cell = pb.cell;
    d.n_slots = e->n_slots;
    d.snap_key = D.snap_key; d.snap_cell_start = D.snap_cell_start; d.snap_sorted = D.snap_sorted;
    d.snap_pair_off = D.snap_pair_off; d.snap_pair_cell = D.snap_pair_cell; d.snap_hdr = D.snap_hdr;
    d.arr_rank = D.arr_rank; d.dep_rank = D.dep_rank; d.arr = D.arr; d.dep = D.dep; d.arr_start = D.arr_start; d.dep_start = D.dep_start;
    d.cnt_enter = D.cnt_enter; d.cnt_leave = D.cnt_leave; d.enter_off = D.enter_off; d.leave_off = D.leave_off;
    d.enter = D.enter; d.leave = D.leave; d.enter_cap = D.enter_cap; d.leave_cap = D.leave_cap;
    d.n_out = D.n_out;
    d.overflow = &e->d_ctr->overflow;
    d.bad_ids = nullptr;
    if (D.ids) {
        // Id mode: the cell CSRs (now: the build's sorted_ent, sorted with d_gid as values; snapshot: its copy) hold global ids, so
        // the kernels must look an entity's cell up by global id.  now_gkey is that lookup for the current state and snap_key, copied
        // from it by the advance, for the snapshot; snap_hdr[0] = n = id_space once a delta has succeeded (0 before: nothing).
        // The kernels treat `e < n ? key[e] : cells` and `ent >= other_n` as "absent"; that stays right because
        //   - every id of a state whose lists are written is < id_space (the scatter checks it, else CHD_OVF_DELTA_IDS);
        //   - an id < id_space that is absent from a state reads 0xFFFFFFFF there, which, like `cells`, no cell list holds;
        //   - an id is in at most one cell (duplicates are refused), as an index is in index mode.
        d.key = D.now_gkey;
        d.n = D.id_space;
        d.bad_ids = D.bad_ids;
        // the CSR by id: sorted_ent, or in entity-table mode (where it holds build positions) the table pass's id-valued copy
        d.sorted = chd_sorted_out(e, c);
    }
    return d;
}

extern "C" {

chd_status chd_delta_on(chd_engine* e, cudaStream_t s) {
    chd_engine::Delta& D = e->dl;
    StageTimer timer(e, s, CHD_STAGE_VISIBLE_DELTA);
    D.n_out = std::max(D.n_out, e->n_slots);
    const DeltaDev d = delta_view(e);
    const uint32_t C = e->g.cells;
    const uint64_t N = e->lim.max_entities;
    chd_status st = chd_epoch_tick(e, s, EP_DELTA);
    if (st != CHD_OK) return st;
    // sizes, the key / pair / cell CSR buffers in use and the ids (the id scatter's, the table lists') are baked into the captured
    // launches
    const EntityIds ids = chd_entity_ids(e);
    uint64_t key = stage_key(0x64656c7461ull, d.n, d.n_slots, D.n_out, e->cur, d.key, d.enter, d.leave, d.enter_cap, d.leave_cap, e->tbl.on,
                             ids.own_ids, ids.gid, ids.own, d.cell_start, d.sorted);  // (the cell CSR: the current copy-input set)
    // id mode: the scatter bakes in the build's length (host count or d_n_build) and the key buffer it reads
    const uint32_t* n_ptr = e->sorted_dev_n ? e->d_n_build : nullptr;
    const uint32_t n_scatter = e->sorted_dev_n ? e->lim.max_entities : e->n_sorted;
    if (D.ids) key = stage_key(key, 0x696473ull, D.id_space, n_scatter, n_ptr, e->d_key, e->d_n_build, d.sorted);
    const unsigned grid = (unsigned)e->sm_count * 8;
    const unsigned slot_grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks_for((uint64_t)D.n_out * 32, DELTA_THREADS), (uint64_t)e->sm_count * 32));
    if (D.read_guard) {  // an asynchronous fetch may still be snapshotting the lists and offsets this delta rewrites
        CU(e, cudaStreamWaitEvent(s, D.ev_read[D.read_fi], 0));
        D.read_guard = false;
    }
    st = run_stage(e, s, D.g, key, [&]() -> chd_status {
        bump_epoch_kernel<<<1, 1, 0, s>>>(e->d_epoch + EP_DELTA);
        KCHECK(e);
        if (D.ids) {
            // The halo import (it writes d_key / d_gid / d_n_build past the own entities) and the build run on the engine stream:
            // a standalone delta follows them there, and a tick's delta (chd_tick_sharded ends in chd_tick) runs on the engine stream
            // after its build or on prep_stream after dl.ev_in, recorded on the engine stream after the build.  Either way the
            // scatter reads this tick's imported halo.
            CU(e, cudaMemsetAsync(D.now_gkey, 0xFF, 4ull * D.id_space, s));
            CU(e, cudaMemsetAsync(D.bad_ids, 0, 4, s));
            delta_id_scatter_kernel<<<grid, DELTA_THREADS, 0, s>>>(ids, e->d_key, n_scatter, n_ptr, C, D.now_gkey, D.id_space, D.bad_ids, d.overflow);
            KCHECK(e);
        }
        SCAN(e, exclusive_scan_fn<DeltaArrivalFlag, uint32_t>(DeltaArrivalFlag{d.sorted, d.key, d.snap_key, d.snap_hdr, d.n, C}, D.arr_rank, N, D.site_arr, s,
                                                              d.cell_start + C));
        SCAN(e, exclusive_scan_fn<DeltaDepartureFlag, uint32_t>(DeltaDepartureFlag{d.snap_sorted, d.snap_key, d.key, d.n, C}, D.dep_rank, N, D.site_dep, s,
                                                                d.snap_cell_start + C));
        delta_moves_kernel<<<grid, DELTA_THREADS, 0, s>>>(d, (uint32_t)N);
        KCHECK(e);
        delta_slots_kernel<false><<<slot_grid, DELTA_THREADS, 0, s>>>(d);
        KCHECK(e);
        SCAN(e, exclusive_scan_1p<uint32_t, uint64_t>(D.cnt_enter, D.enter_off, D.n_out, D.site_enter, s));
        SCAN(e, exclusive_scan_1p<uint32_t, uint64_t>(D.cnt_leave, D.leave_off, D.n_out, D.site_leave, s));
        delta_slots_kernel<true><<<slot_grid, DELTA_THREADS, 0, s>>>(d);
        KCHECK(e);
        if (e->tbl.on && !D.ids) {  // entity-table index mode: the lists name ids (here: a later spawn must not change lists already computed)
            const chd_status ts = chd_table_delta_ids(e, s);
            if (ts != CHD_OK) return ts;
        }
        delta_advance_kernel<<<grid, DELTA_THREADS, 0, s>>>(d, (uint32_t)e->lim.max_pairs);
        KCHECK(e);
        return CHD_OK;
    });
    if (st != CHD_OK) return st;
    CU(e, cudaEventRecord(D.ev_end, s));
    D.seq++;
    return CHD_OK;
}

// The first reserve picks the mode (ids: id mode over [0, id_space)) and allocates; every later one only grows the lists.
static chd_status delta_reserve(chd_engine* e, uint64_t cap_entries, bool ids, uint32_t id_space) {
    // a delta of an earlier tick may still be running (on the engine stream or, inside a tick, on prep_stream)
    CU(e, cudaStreamSynchronize(e->stream));
    CU(e, cudaStreamSynchronize(e->prep_stream));
    // an asynchronous fetch may still be snapshotting the lists that ensure_cap frees
    if (e->dl_stream_d) CU(e, cudaStreamSynchronize(e->dl_stream_d));
    chd_engine::Delta& D = e->dl;
    const uint64_t N = e->lim.max_entities, S = e->lim.max_subscribers, P = e->lim.max_pairs, C = e->g.cells;
    if (!D.on) {
        // id mode: snap_key and now_gkey are indexed by global id
        const bool ok = dalloc(e, &D.snap_key, ids ? (uint64_t)id_space : N) &&
                        (!ids || (dalloc(e, &D.now_gkey, id_space) && dalloc(e, &D.bad_ids, 1))) && dalloc(e, &D.snap_cell_start, C + 2) &&
                        dalloc(e, &D.snap_sorted, N) &&
                        dalloc(e, &D.snap_pair_off, S + 1) && dalloc(e, &D.snap_pair_cell, P) && dalloc(e, &D.snap_hdr, 2) &&
                        dalloc(e, &D.arr_rank, N + 1) && dalloc(e, &D.dep_rank, N + 1) && dalloc(e, &D.arr, N) && dalloc(e, &D.dep, N) &&
                        dalloc(e, &D.arr_start, C + 1) && dalloc(e, &D.dep_start, C + 1) && dalloc(e, &D.cnt_enter, S) &&
                        dalloc(e, &D.cnt_leave, S) && dalloc(e, &D.enter_off, S + 1) && dalloc(e, &D.leave_off, S + 1) &&
                        chd_make_site(e, D.site_arr, N + 1, EP_DELTA) && chd_make_site(e, D.site_dep, N + 1, EP_DELTA) &&
                        chd_make_site(e, D.site_enter, S + 1, EP_DELTA) && chd_make_site(e, D.site_leave, S + 1, EP_DELTA) &&
                        chd_make_event(e, &D.ev_in) && chd_make_event(e, &D.ev_done) && chd_make_event(e, &D.ev_end) &&
                        chd_make_event(e, &D.ev_read[0]) && chd_make_event(e, &D.ev_read[1]);
        if (!ok) return CHD_ERR_CUDA;
        for (ScanSite* site : {&D.site_arr, &D.site_dep, &D.site_enter, &D.site_leave}) site->error = &e->d_ctr->overflow;
        // the empty snapshot: no entities, no cells populated, no slots
        CU(e, cudaMemsetAsync(D.snap_hdr, 0, 8, e->stream));
        CU(e, cudaMemsetAsync(D.snap_cell_start, 0, (C + 2) * 4, e->stream));
        CU(e, cudaMemsetAsync(D.snap_pair_off, 0, (S + 1) * 4, e->stream));
        CU(e, cudaStreamSynchronize(0));  // (chd_make_site clears its descriptors on the default stream)
        D.on = true;
        D.ids = ids;
        D.id_space = ids ? id_space : 0;
    }
    if (!ensure_cap(e, &D.enter, &D.enter_cap, cap_entries, cap_entries) || !ensure_cap(e, &D.leave, &D.leave_cap, cap_entries, cap_entries))
        return CHD_ERR_CUDA;
    // the lists of the last delta are gone (a grown buffer starts empty): report an empty delta until the next one
    CU(e, cudaMemsetAsync(D.enter_off, 0, (S + 1) * 8, e->stream));
    CU(e, cudaMemsetAsync(D.leave_off, 0, (S + 1) * 8, e->stream));
    if (D.ids) CU(e, cudaMemsetAsync(D.bad_ids, 0, 4, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

chd_status chd_reserve_visible_delta(chd_engine* e, uint64_t cap_entries) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_index_delta(e) != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    return delta_reserve(e, cap_entries, e->dl.ids, e->dl.id_space);  // (id mode: grows the lists only)
}

chd_status chd_reserve_visible_delta_ids(chd_engine* e, uint64_t cap_entries, uint32_t id_space) {
    if (!e || id_space == 0) return CHD_ERR_INVALID;
    const chd_status st = chd_rule_id_delta(e, id_space);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return delta_reserve(e, cap_entries, true, id_space);
}

chd_status chd_visible_delta(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_delta_check(e, false) != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_FETCH_GUARD);
    return chd_delta_on(e, e->stream);
}

chd_status chd_read_delta_lengths(chd_engine* e, cudaStream_t s, DeltaLengths* out) {
    const chd_engine::Delta& D = e->dl;
    uint64_t* h64 = (uint64_t*)e->h_get;
    h64[2] = 0;
    CU(e, cudaMemcpyAsync(h64, D.enter_off + D.n_out, 8, cudaMemcpyDeviceToHost, s));
    CU(e, cudaMemcpyAsync(h64 + 1, D.leave_off + D.n_out, 8, cudaMemcpyDeviceToHost, s));
    if (D.ids) CU(e, cudaMemcpyAsync(h64 + 2, D.bad_ids, 4, cudaMemcpyDeviceToHost, s));
    CU(e, cudaStreamSynchronize(s));
    *out = DeltaLengths{h64[0], h64[1], (uint32_t)h64[2] != 0};
    return CHD_OK;
}

chd_status chd_get_visible_delta(chd_engine* e, uint64_t* enter_off, uint32_t* enter_entity, uint64_t* leave_off, uint32_t* leave_entity,
                                 uint64_t cap, uint64_t* n_entered, uint64_t* n_left, uint32_t* n_slots) {
    if (!e) return CHD_ERR_INVALID;
    chd_engine::Delta& D = e->dl;
    if (!D.on) {
        e->fail("chd_get_visible_delta before chd_reserve_visible_delta");
        return CHD_ERR_STATE;
    }
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    cudaStream_t s = e->stream;  // (a tick's delta on prep_stream is joined into the engine stream)
    const uint32_t S = D.n_out;
    DeltaLengths dn;
    const chd_status st = chd_read_delta_lengths(e, s, &dn);
    if (st != CHD_OK) return st;
    const uint64_t ne = dn.n_entered, nl = dn.n_left;
    if (n_entered) *n_entered = ne;
    if (n_left) *n_left = nl;
    if (n_slots) *n_slots = S;
    if (enter_off) CU(e, cudaMemcpyAsync(enter_off, D.enter_off, 8ull * (S + 1ull), cudaMemcpyDefault, s));
    if (leave_off) CU(e, cudaMemcpyAsync(leave_off, D.leave_off, 8ull * (S + 1ull), cudaMemcpyDefault, s));
    if (enter_entity || leave_entity) {
        if (chd_delta_overflowed(ne, nl, D.enter_cap, D.leave_cap, dn.bad_ids)) {
            CU(e, cudaStreamSynchronize(s));
            if (dn.bad_ids) {
                e->fail("the last visible delta met an id >= id_space %u or an id held twice (CHD_OVF_DELTA_IDS): no lists", D.id_space);
                return CHD_ERR_INVALID;
            }
            e->fail("the last visible delta overflowed (CHD_OVF_DELTA): %llu entered / %llu left > capacity %llu",
                    (unsigned long long)ne, (unsigned long long)nl, (unsigned long long)std::min(D.enter_cap, D.leave_cap));
            return CHD_ERR_CAPACITY;
        }
        if ((enter_entity && ne > cap) || (leave_entity && nl > cap)) {
            CU(e, cudaStreamSynchronize(s));
            e->fail("chd_get_visible_delta: %llu entered / %llu left > cap %llu", (unsigned long long)ne, (unsigned long long)nl,
                    (unsigned long long)cap);
            return CHD_ERR_CAPACITY;
        }
        if (enter_entity && ne) CU(e, cudaMemcpyAsync(enter_entity, D.enter, 4ull * ne, cudaMemcpyDefault, s));
        if (leave_entity && nl) CU(e, cudaMemcpyAsync(leave_entity, D.leave, 4ull * nl, cudaMemcpyDefault, s));
    }
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}
}  // extern "C"
