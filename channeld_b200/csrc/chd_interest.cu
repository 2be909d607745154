// chd_interest.cu — subscribers, SpatialInterestQuery batches, QueryChannelIds (stateless) and the interest update
// (handleUpdateSpatialInterest, batched).
#include "chd_engine.h"

#include "chd_interest.cuh"
#include "chd_misc.cuh"

extern "C" {

chd_status chd_prefetch_queries(chd_engine* e, const chd_query_batch* q) {
    if (!e || !q) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    int set = 0;
    chd_status st = chd_pf_begin(e, e->pf_q, &set);
    if (st != CHD_OK) return st;
    chd_engine::QStage& qs = e->dq_pf[set];
    if (!qs.spot_dist && !alloc_qstage(e, qs)) return CHD_ERR_CUDA;  // (spot_dist is allocated last)
    st = chd_upload_queries(e, e->up_stream, q, &qs.view, true, &qs, &qs.spots);
    return st != CHD_OK ? st : chd_pf_end(e, e->pf_q);
}

/* ------------------------------------------------------------------ subscribers / queries ---- */

chd_status chd_set_subscribers(chd_engine* e, const uint32_t* conn_id, uint32_t n) {
    if (!e || (n && !conn_id)) return CHD_ERR_INVALID;
    if (n > e->lim.max_subscribers) {
        e->fail("chd_set_subscribers: %u > max_subscribers %u", n, e->lim.max_subscribers);
        return CHD_ERR_CAPACITY;
    }
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaMemcpyAsync(e->d_conn, conn_id, sizeof(uint32_t) * n, cudaMemcpyDefault, e->stream));
    CU(e, cudaMemsetAsync(e->pairs[0].off, 0, ((uint64_t)e->lim.max_subscribers + 1) * 4, e->stream));
    CU(e, cudaMemsetAsync(e->pairs[1].off, 0, ((uint64_t)e->lim.max_subscribers + 1) * 4, e->stream));
    CU(e, cudaMemsetAsync(e->d_vis_off, 0, ((uint64_t)e->lim.max_subscribers + 1) * 8, e->stream));
    CU(e, cudaMemsetAsync(e->d_slot_ctl, 0, e->lim.max_subscribers, e->stream));
    if (n < e->lim.max_subscribers) CU(e, cudaMemsetAsync(e->d_conn + n, 0, sizeof(uint32_t) * (e->lim.max_subscribers - n), e->stream));
    e->n_slots = n;
    e->cur = 0;
    return chd_follow_drop(e, nullptr, nullptr, 0);  // no slot follows an entity any more
}

// slots (+ an optional per-slot value) of a lifecycle call -> device staging; slot lists are control-plane sized
static chd_status upload_slot_list(chd_engine* e, const uint32_t* slot, const uint32_t* aux, uint32_t n, uint32_t* max_slot) {
    if (n > e->lim.max_subscribers) {
        e->fail("lifecycle call with %u slots > max_subscribers %u", n, e->lim.max_subscribers);
        return CHD_ERR_CAPACITY;
    }
    *max_slot = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (slot[i] >= e->lim.max_subscribers) {
            e->fail("slot %u >= max_subscribers %u", slot[i], e->lim.max_subscribers);
            return CHD_ERR_INVALID;
        }
        if (slot[i] > *max_slot) *max_slot = slot[i];
    }
    // the host arrays are plain pageable memory in general: a synchronous copy keeps the cgo pointer rules trivially true
    CU(e, cudaMemcpyAsync(e->d_lc_slot, slot, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, e->stream));
    if (aux) CU(e, cudaMemcpyAsync(e->d_lc_aux, aux, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

chd_status chd_grow_slots(chd_engine* e, uint32_t new_n) {
    if (new_n <= e->n_slots) return CHD_OK;
    CU(e, chd_copy_wait(e));  // only when the table grows: the copy kernel reads the pair offsets
    const uint32_t old_n = e->n_slots;
    extend_offsets_kernel<<<blocks_for(new_n - old_n, 256), 256, 0, e->stream>>>(e->pairs[e->cur].off, old_n, new_n);
    KCHECK(e);
    CU(e, cudaMemsetAsync(e->d_vis_off + old_n + 1, 0, sizeof(uint64_t) * (new_n - old_n), e->stream));  // refreshed by the next emit
    e->n_slots = new_n;
    return CHD_OK;
}

chd_status chd_add_subscribers(chd_engine* e, const uint32_t* slot, const uint32_t* conn_id, uint32_t n) {
    if (!e || (n && (!slot || !conn_id))) return CHD_ERR_INVALID;
    if (n == 0) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    uint32_t max_slot = 0;
    chd_status st = upload_slot_list(e, slot, conn_id, n, &max_slot);
    if (st != CHD_OK) return st;
    slot_ctl_set_kernel<<<blocks_for(n, 256), 256, 0, e->stream>>>(e->d_lc_slot, e->d_lc_aux, n, (uint8_t)SLOT_NORMAL, 0u, e->d_slot_ctl, e->d_slot_src, e->d_conn);
    KCHECK(e);
    st = chd_grow_slots(e, max_slot + 1);
    if (st != CHD_OK) return st;
    e->lifecycle_used = true;
    return CHD_OK;
}

chd_status chd_remove_subscribers(chd_engine* e, const uint32_t* slot, uint32_t n) {
    if (!e || (n && !slot)) return CHD_ERR_INVALID;
    if (n == 0) return CHD_OK;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    uint32_t max_slot = 0;
    chd_status st = upload_slot_list(e, slot, nullptr, n, &max_slot);
    if (st != CHD_OK) return st;
    if (max_slot >= e->n_slots) {
        e->fail("chd_remove_subscribers: slot %u is not in use (%u slots)", max_slot, e->n_slots);
        return CHD_ERR_INVALID;
    }
    slot_ctl_set_kernel<<<blocks_for(n, 256), 256, 0, e->stream>>>(e->d_lc_slot, nullptr, n, (uint8_t)SLOT_REMOVE, 0u, e->d_slot_ctl, e->d_slot_src, nullptr);
    KCHECK(e);
    e->lifecycle_used = true;
    return chd_follow_drop(e, slot, e->d_lc_slot, n);  // a removed slot follows nothing
}

chd_status chd_upload_queries(chd_engine* e, cudaStream_t s, const chd_query_batch* q, QueryDev* out, bool need_sub, chd_engine::QStage* stage,
                              uint32_t* spots) {
    if (!q) return CHD_ERR_INVALID;
    chd_engine::QStage& dq = stage ? *stage : e->dq;
    const uint32_t n = q->n;
    if (n > e->lim.max_queries) {
        e->fail("query batch of %u > max_queries %u", n, e->lim.max_queries);
        return CHD_ERR_CAPACITY;
    }
    QueryDev d{};
    d.n = n;
    if (spots) *spots = 0;
#define UP(field, T)                                                                                      \
    if (q->field) {                                                                                       \
        if (chd_is_device_ptr(e, q->field)) {                                                                 \
            d.field = q->field; /* device-resident batch: consumed in place */                            \
        } else {                                                                                          \
            CU(e, cudaMemcpyAsync(dq.field, q->field, sizeof(T) * n, cudaMemcpyDefault, s));           \
            d.field = dq.field;                                                                        \
        }                                                                                                 \
    }
    if (need_sub) {
        if (!q->sub && n > e->n_slots) {
            e->fail("identity query batch (sub == NULL) of %u queries > %u subscribers", n, e->n_slots);
            return CHD_ERR_INVALID;
        }
        UP(sub, uint32_t);
    }
    UP(kind, uint8_t);
    UP(sph_cx, double); UP(sph_cz, double); UP(sph_r, double);
    UP(box_cx, double); UP(box_cz, double); UP(box_ex, double); UP(box_ez, double);
    UP(cone_cx, double); UP(cone_cz, double); UP(cone_dx, double); UP(cone_dz, double); UP(cone_angle, double); UP(cone_r, double);
    UP(spot_ndist, uint32_t);
#undef UP
    if (!q->kind && n && (!q->sph_cx || !q->sph_cz || !q->sph_r)) {
        e->fail("kind == NULL means all-sphere: sph_cx/sph_cz/sph_r are required");
        return CHD_ERR_INVALID;
    }
    if (q->spot_off) {
        // spot_off may live on the host or on the device; its last element sizes the spot arrays
        uint32_t total = 0;
        CU(e, cudaMemcpyAsync(dq.spot_off, q->spot_off, sizeof(uint32_t) * ((uint64_t)n + 1), cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(e->h_u32, dq.spot_off + n, 4, cudaMemcpyDeviceToHost, s));
        CU(e, cudaStreamSynchronize(s));
        total = *e->h_u32;
        if (spots) *spots = total;
        if (total > e->lim.max_spots) {
            e->fail("%u spots > max_spots %u", total, e->lim.max_spots);
            return CHD_ERR_CAPACITY;
        }
        if (total && (!q->spot_x || !q->spot_z)) return CHD_ERR_INVALID;
        CU(e, cudaMemcpyAsync(dq.spot_x, q->spot_x, sizeof(double) * total, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(dq.spot_z, q->spot_z, sizeof(double) * total, cudaMemcpyDefault, s));
        if (q->spot_dist) CU(e, cudaMemcpyAsync(dq.spot_dist, q->spot_dist, sizeof(uint32_t) * total, cudaMemcpyDefault, s));
        else CU(e, cudaMemsetAsync(dq.spot_dist, 0, sizeof(uint32_t) * total, s));
        d.spot_off = dq.spot_off; d.spot_x = dq.spot_x; d.spot_z = dq.spot_z; d.spot_dist = dq.spot_dist;
        if (!q->spot_ndist) {
            CU(e, cudaMemsetAsync(dq.spot_ndist, 0, sizeof(uint32_t) * n, s));
            d.spot_ndist = dq.spot_ndist;
        }
    }
    *out = d;
    return CHD_OK;
}

// Q1 + scan + Q2: fills bbox / window / side lists / status / qcount for the batch
// bounding box -> window scratch -> lattice walk, one launch: fills bbox / window / side lists / status / qcount for the batch.
// The caller has zeroed the window cursor (stage_begin_kernel / a memset on the stateless path).
static chd_status run_query_kernel(chd_engine* e, cudaStream_t s, const QueryDev& d, uint32_t* status) {
    const uint32_t n = d.n;
    if (n == 0) return CHD_OK;
    query_kernel<<<blocks_for(n, 128), 128, 0, s>>>(e->g, d, e->d_bbox, e->d_win_off, e->lim.max_window_cells, e->d_win_cursor, e->d_window,
                                                    e->d_side_cell, e->d_side_dist, e->d_side_cnt, status, e->d_qcount, &e->d_ctr->overflow);
    KCHECK(e);
    return CHD_OK;
}

chd_status chd_query_channel_ids(chd_engine* e, const chd_query_batch* q, uint32_t* out_status, uint32_t* out_off,
                                 uint32_t* out_channel_id, uint32_t* out_dist, uint64_t cap) {
    if (!e || !q) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    CU(e, cudaStreamSynchronize(e->aux_stream));  // an in-flight interest update shares the query scratch
    QueryDev d;
    chd_status st = chd_upload_queries(e, e->stream, q, &d, false);
    if (st != CHD_OK) return st;
    const uint32_t n = d.n;
    if (n == 0) {
        if (out_off) {
            const uint32_t zero = 0;
            CU(e, cudaMemcpyAsync(out_off, &zero, 4, cudaMemcpyDefault, e->stream));
            CU(e, cudaStreamSynchronize(e->stream));
        }
        return CHD_OK;
    }
    // own status array: the statuses of the last interest batch (chd_get_query_status / chd_fetch_results) are not disturbed
    chd_epoch_tick(e, e->stream, EP_QUERY);
    bump_epoch_kernel<<<1, 1, 0, e->stream>>>(e->d_epoch + EP_QUERY);
    KCHECK(e);
    CU(e, cudaMemsetAsync(e->d_win_cursor, 0, 8, e->stream));
    st = run_query_kernel(e, e->stream, d, e->d_qstatus);
    if (st != CHD_OK) return st;
    SCAN(e, exclusive_scan_1p<uint32_t, uint64_t>(e->d_qcount, e->d_qoff, n, e->site_qoff, e->stream));
    const uint64_t dev_cap = e->lim.max_pairs;
    query_write_kernel<<<blocks_for(n, 128), 128, 0, e->stream>>>(e->g, n, e->d_qstatus, e->d_bbox, e->d_win_off, e->d_window, e->d_side_cell,
                                                                  e->d_side_dist, e->d_side_cnt, d.spot_off, e->d_qoff, dev_cap,
                                                                  e->d_qout_id, e->d_qout_dist);
    KCHECK(e);
    // totals
    uint64_t* h64 = (uint64_t*)e->h_u32;
    CU(e, cudaMemcpyAsync(h64, e->d_qoff + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaMemcpyAsync(h64 + 1, e->d_win_cursor, 8, cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    const uint64_t total = h64[0], wtotal = h64[1];
    if (wtotal > e->lim.max_window_cells) {  // some queries got CHD_Q_ERR_CAPACITY: report the batch as a capacity failure
        e->fail("query windows need %llu cells > max_window_cells %llu", (unsigned long long)wtotal,
                (unsigned long long)e->lim.max_window_cells);
        CU(e, cudaMemsetAsync(&e->d_ctr->overflow, 0, 4, e->stream));  // (the stateless path reports through its return value)
        return CHD_ERR_CAPACITY;
    }
    if (total > dev_cap || total > cap) {
        e->fail("query result has %llu entries > capacity %llu", (unsigned long long)total,
                (unsigned long long)(total > dev_cap ? dev_cap : cap));
        return CHD_ERR_CAPACITY;
    }
    if (out_status) CU(e, cudaMemcpyAsync(out_status, e->d_qstatus, sizeof(uint32_t) * n, cudaMemcpyDefault, e->stream));
    if (out_off) {
        // u64 device offsets -> u32 caller offsets
        narrow_offsets_kernel<<<blocks_for((uint64_t)n + 1, 256), 256, 0, e->stream>>>(e->d_qoff, n + 1, e->d_new_off);
        KCHECK(e);
        CU(e, cudaMemcpyAsync(out_off, e->d_new_off, sizeof(uint32_t) * ((uint64_t)n + 1), cudaMemcpyDefault, e->stream));
    }
    if (out_channel_id) CU(e, cudaMemcpyAsync(out_channel_id, e->d_qout_id, sizeof(uint32_t) * total, cudaMemcpyDefault, e->stream));
    if (out_dist) CU(e, cudaMemcpyAsync(out_dist, e->d_qout_dist, sizeof(uint32_t) * total, cudaMemcpyDefault, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

// part 0: query -> new subscription pairs (everything emit needs); part 1: pairs grouped by cell + diff lists
// (needed by the fan-out pass and the host only).  An event between the two lets emit start early.
static chd_status interest_enqueue(chd_engine* e, cudaStream_t s, const QueryDev& d, int part) {
    const uint32_t n = d.n, S = e->n_slots;
    chd_status st = CHD_OK;
    PairBuf& prev = e->pairs[e->cur];
    PairBuf& cur = e->pairs[e->cur ^ 1];
    const uint64_t P = e->lim.max_pairs;
    if (part == 0) {
    st = run_query_kernel(e, s, d, e->d_status);
    if (st != CHD_OK) return st;
    // sub == NULL is the identity batch (query i <-> subscriber slot i): no slot table needed
    const int32_t* slot_query = d.sub ? e->d_slot_query : nullptr;
    if (d.sub) CU(e, cudaMemsetAsync(e->d_slot_query, 0xFF, sizeof(int32_t) * (uint64_t)(S ? S : 1), s));
    if (n && d.sub) {
        slot_scatter_kernel<<<blocks_for(n, 256), 256, 0, s>>>(d.sub, n, S, e->d_slot_query);
        KCHECK(e);
    }
    const uint8_t* ctl_in = e->lifecycle_used ? e->d_slot_ctl : nullptr;
    SCAN(e, exclusive_scan_fn<SlotCountIn, uint32_t>(SlotCountIn{slot_query, n, e->d_status, e->d_qcount, prev, ctl_in, e->d_slot_src, e->mig}, e->d_noff, S,
                                                     e->site_slot, s));
    if (S) {
        interest_fill_kernel<<<blocks_for(S, 128), 128, 0, s>>>(e->g, S, slot_query, n, e->d_status, e->d_bbox, e->d_win_off, e->d_window,
                                                                e->d_side_cell, e->d_side_dist, e->d_side_cnt, d.spot_off, prev, cur, e->d_noff, P,
                                                                e->d_time, DiffOut{e->d_new_sub, e->d_new_ch, e->d_gone_sub, e->d_gone_ch}, e->d_pair_ch, e->d_win_cursor,
                                                                e->d_ctr, e->lifecycle_used ? e->d_slot_ctl : nullptr, e->d_slot_src, e->d_conn, e->mig,
                                                                e->have_cell_start ? e->d_cell_start_ns : nullptr, e->d_cell_max_interval);
        e->pair_ch_valid = true;
        e->by_cell_valid = true;
        KCHECK(e);
    }
    return CHD_OK;
    }  // part 0
    // pairs grouped by cell for the fan-out pass (= every channel's subscriber list): a stable radix sort of pair indices by cell
    // (cells are in [0, C)) with the same kernels as the entity build (no global atomics), device-side length
    return chd_cell_sort(e, s, e->pair_sort, e->g.cells, cur.cell, nullptr, (uint32_t)P, cur.off + S, nullptr, e->d_by_cell);
}

chd_status chd_update_interest(chd_engine* e, const chd_query_batch* q, int64_t now_ns) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_rings_staged(e, "chd_update_interest") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD);
    return chd_update_interest_on(e, e->stream, q, now_ns);
}

chd_status chd_update_interest_on(chd_engine* e, cudaStream_t s, const chd_query_batch* q, int64_t now_ns) {
    std::lock_guard<std::recursive_mutex> lk(e->mu);  // the query scratch
    StageTimer timer(e, s, CHD_STAGE_INTEREST);
    QueryDev d;
    chd_status st;
    int pf_set = -1;  // prefetch staging set this batch lives in
    if (!q && e->fw.ready) {  // the batch generated by chd_follow_queries: device-resident, ordered before this on the engine stream
        d = e->fw.view;
        e->fw.ready = false;  // consumed
    } else if (!q) {  // the batch uploaded by chd_prefetch_queries and handed over by chd_adopt_prefetched
        if (e->pf_q.cur < 0) {
            e->fail("interest update without a batch: q == NULL needs chd_prefetch_queries + chd_adopt_prefetched, or chd_follow_queries, first");
            return CHD_ERR_STATE;
        }
        pf_set = e->pf_q.cur;
        d = e->dq_pf[pf_set].view;
        e->pf_q.cur = -1;  // consumed
        if (d.n > e->n_slots && !d.sub) {
            e->fail("identity query batch (sub == NULL) of %u queries > %u subscribers", d.n, e->n_slots);
            return CHD_ERR_INVALID;
        }
        st = chd_pf_wait(e, e->pf_q, s);
        if (st != CHD_OK) return st;
    } else {
        st = chd_upload_queries(e, s, q, &d, true);  // H2D / D2D copies into the engine's SoA: outside the graph
        if (st != CHD_OK) return st;
    }
    // (outside the replayed graphs: the tick time is a launch argument) tick time, new scan epoch, zeroed counters
    // n_query_errors / n_sub_new / n_unsub / n_kept and window cursor
    chd_epoch_tick(e, s, EP_QUERY);
    stage_begin_kernel<<<1, 1, 0, s>>>(e->d_time, now_ns, e->d_epoch + EP_QUERY, &e->d_ctr->n_query_errors, 4, e->d_win_cursor);
    KCHECK(e);
    // the graph bakes in which staging arrays are live, the batch size and the pair-buffer parity
    const uint64_t key = stage_key(0x696e74ull, d.n, e->n_slots, e->cur, e->lifecycle_used, e->mig.base, e->have_cell_start, d.sub, d.kind, d.sph_cx,
                                   d.sph_cz, d.sph_r, d.box_cx, d.box_cz, d.box_ex, d.box_ez, d.cone_cx, d.cone_cz, d.cone_dx, d.cone_dz, d.cone_angle,
                                   d.cone_r, d.spot_off, d.spot_ndist, d.spot_x, d.spot_z, d.spot_dist, d.missing);
    st = run_stage(e, s, e->g_interest, key, [&]() { return interest_enqueue(e, s, d, 0); });
    if (st != CHD_OK) return st;
    CU(e, cudaEventRecord(e->ev_pairs, s));  // the new pairs exist: emit may start (chd_tick waits on this)
    st = run_stage(e, s, e->g_interest_b, stage_key(key, 0xb), [&]() { return interest_enqueue(e, s, d, 1); });
    if (st != CHD_OK) return st;
    st = chd_pf_note_read(e, e->pf_q, pf_set, s);  // the staging set may be refilled once these kernels have run
    if (st != CHD_OK) return st;
    e->cur ^= 1;
    e->last_nq = d.n;
    return CHD_OK;
}
}  // extern "C"
