// chd_extras.cu — rows of SURVEY.md §8f built on the tick's results (window classes of the due list, ADJACENT_CHANNELS
// broadcast sets) and the config-plane helpers of the SpatialController surface.
#include "chd_engine.h"

#include "chd_broadcast.cuh"
#include "chd_classes.cuh"

extern "C" {

/* ------------------------------------------------------------------ window classes of the due list ---- */

chd_status chd_due_classes(chd_engine* e, uint32_t* out_class_of, uint32_t* out_class_rep, uint32_t* out_class_count, uint32_t cap_classes,
                           uint32_t* out_n_classes) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    cudaStream_t s = e->stream;
    uint32_t n_due = 0;
    chd_status st = chd_read_u32(e, &e->d_ctr->n_due, &n_due);
    if (st != CHD_OK) return st;
    if (n_due > e->lim.max_due) n_due = e->lim.max_due;
    if (out_n_classes) *out_n_classes = 0;
    if (n_due == 0) return CHD_OK;
    const uint64_t D = e->lim.max_due;
    if (!e->d_cls_table) {
        uint32_t T = 1024;
        while ((uint64_t)T < 2 * D) T <<= 1;
        if (!(dalloc(e, &e->d_cls_table, (uint64_t)T) && dalloc(e, &e->d_cls_rep, (uint64_t)T) && dalloc(e, &e->d_cls_cnt, (uint64_t)T) &&
              dalloc(e, &e->d_cls_slot, D) && dalloc(e, &e->d_cls_flag, D + 1) && dalloc(e, &e->d_cls_rank, D + 1) && dalloc(e, &e->d_cls_of, D) &&
              dalloc(e, &e->d_cls_out_rep, D) && dalloc(e, &e->d_cls_out_cnt, D) && chd_make_site(e, e->site_class, D + 1, EP_CLASS)))
            return CHD_ERR_CUDA;
        e->site_class.error = &e->d_ctr->overflow;
        e->cls_table_size = T;
    }
    // a table of >= 2 n slots is enough for this call: clear only that much
    uint32_t T = 1024;
    while ((uint64_t)T < 2ull * n_due) T <<= 1;
    CU(e, cudaMemsetAsync(e->d_cls_table, 0xFF, 4ull * T, s));
    CU(e, cudaMemsetAsync(e->d_cls_rep, 0xFF, 4ull * T, s));
    CU(e, cudaMemsetAsync(e->d_cls_cnt, 0, 4ull * T, s));
    const uint32_t* n_ptr = &e->d_ctr->n_due;
    st = chd_epoch_tick(e, s, EP_CLASS);
    if (st != CHD_OK) return st;
    const unsigned blocks = blocks_for(n_due, 256);
    class_insert_kernel<<<blocks, 256, 0, s>>>(e->d_due, e->d_due_key, n_ptr, e->lim.max_due, e->d_cls_table, T - 1, e->d_cls_slot, e->d_cls_rep,
                                               e->d_cls_cnt);
    KCHECK(e);
    class_flag_kernel<<<blocks, 256, 0, s>>>(n_ptr, e->lim.max_due, e->d_cls_slot, e->d_cls_rep, e->d_cls_flag, e->d_epoch + EP_CLASS);
    KCHECK(e);
    SCAN(e, exclusive_scan_1p<uint32_t, uint32_t>(e->d_cls_flag, e->d_cls_rank, n_due, e->site_class, s));
    class_finish_kernel<<<blocks, 256, 0, s>>>(n_ptr, e->lim.max_due, e->d_cls_slot, e->d_cls_rep, e->d_cls_cnt, e->d_cls_rank, e->d_cls_of,
                                               e->d_cls_out_rep, e->d_cls_out_cnt);
    KCHECK(e);
    uint32_t n_classes = 0;
    st = chd_read_u32(e, e->d_cls_rank + n_due, &n_classes);
    if (st != CHD_OK) return st;
    if (out_n_classes) *out_n_classes = n_classes;
    if ((out_class_rep || out_class_count) && n_classes > cap_classes) {
        e->fail("chd_due_classes: %u classes > cap_classes %u", n_classes, cap_classes);
        return CHD_ERR_CAPACITY;
    }
    if (out_class_of) CU(e, cudaMemcpyAsync(out_class_of, e->d_cls_of, 4ull * n_due, cudaMemcpyDefault, s));
    if (out_class_rep) CU(e, cudaMemcpyAsync(out_class_rep, e->d_cls_out_rep, 4ull * n_classes, cudaMemcpyDefault, s));
    if (out_class_count) CU(e, cudaMemcpyAsync(out_class_count, e->d_cls_out_cnt, 4ull * n_classes, cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

/* ------------------------------------------------------------------ ADJACENT_CHANNELS broadcast sets ---- */

__global__ void bcast_msgoff_kernel(const uint32_t* __restrict__ off9, uint32_t n, uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n) out[i] = off9[(uint64_t)i * 9];
}

chd_status chd_set_subscriber_types(chd_engine* e, const uint8_t* conn_type, uint32_t n) {
    if (!e || n > e->lim.max_subscribers) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    if (!conn_type) {
        e->have_conn_type = false;
        return CHD_OK;
    }
    if (!e->d_conn_type && !dalloc(e, &e->d_conn_type, (uint64_t)e->lim.max_subscribers)) return CHD_ERR_CUDA;
    CU(e, cudaMemsetAsync(e->d_conn_type, 0, e->lim.max_subscribers, e->stream));
    CU(e, cudaMemcpyAsync(e->d_conn_type, conn_type, n, cudaMemcpyDefault, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    e->have_conn_type = true;
    return CHD_OK;
}

chd_status chd_adjacent_broadcast(chd_engine* e, const chd_broadcast_batch* b, uint32_t* out_status, uint32_t* out_off, uint32_t* out_slot,
                                  uint64_t cap) {
    if (!e || !b || (b->n && (!b->channel_id || !b->broadcast)) || !out_off) return CHD_ERR_INVALID;
    if (chd_rule_no_chain(e, "chd_adjacent_broadcast", false) != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_COPY_WAIT);
    const uint32_t n = b->n;
    if (out_status)
        for (uint32_t m = 0; m < n; m++)
            out_status[m] = (b->channel_id[m] >= e->g.id_start && b->channel_id[m] - e->g.id_start < e->g.cells) ? CHD_BC_OK : CHD_BC_ERR_NOT_A_CELL;
    if (n == 0 || !e->by_cell_valid || e->n_slots == 0) {  // no messages, or nobody is subscribed to anything yet
        for (uint32_t m = 0; m <= n; m++) out_off[m] = 0;
        return CHD_OK;
    }
    cudaStream_t s = e->stream;
    CU(e, cudaStreamSynchronize(e->aux_stream));  // an interest update in flight is rewriting the pairs / by-cell order
    if (n > e->bc_msg_cap) {
        const uint64_t c = std::max<uint64_t>(1024, (uint64_t)n + n / 2);
        chd_dfree(e, e->d_bc_in); chd_dfree(e, e->d_bc_cnt); chd_dfree(e, e->d_bc_off); chd_dfree(e, e->d_bc_msgoff); chd_dfree(e, e->site_bcast.desc);
        e->d_bc_in = e->d_bc_cnt = e->d_bc_off = e->d_bc_msgoff = nullptr;
        e->site_bcast.desc = nullptr;
        e->bc_msg_cap = 0;
        if (!dalloc(e, &e->d_bc_in, 4 * c) || !dalloc(e, &e->d_bc_cnt, 9 * c + 1) || !dalloc(e, &e->d_bc_off, 9 * c + 1) ||
            !dalloc(e, &e->d_bc_msgoff, c + 1) || !chd_make_site(e, e->site_bcast, 9 * c + 1, EP_BCAST))
            return CHD_ERR_CUDA;
        e->site_bcast.error = &e->d_ctr->overflow;
        e->bc_msg_cap = c;
    }
    const uint64_t mc = e->bc_msg_cap;
    CU(e, cudaMemcpyAsync(e->d_bc_in, b->channel_id, 4ull * n, cudaMemcpyDefault, s));
    CU(e, cudaMemcpyAsync(e->d_bc_in + mc, b->broadcast, 4ull * n, cudaMemcpyDefault, s));
    if (b->sender_conn_id) CU(e, cudaMemcpyAsync(e->d_bc_in + 2 * mc, b->sender_conn_id, 4ull * n, cudaMemcpyDefault, s));
    else CU(e, cudaMemsetAsync(e->d_bc_in + 2 * mc, 0, 4ull * n, s));
    if (b->client_conn_id) CU(e, cudaMemcpyAsync(e->d_bc_in + 3 * mc, b->client_conn_id, 4ull * n, cudaMemcpyDefault, s));
    else CU(e, cudaMemsetAsync(e->d_bc_in + 3 * mc, 0, 4ull * n, s));
    const BcastDev bd{n, e->d_bc_in, e->d_bc_in + mc, e->d_bc_in + 2 * mc, e->d_bc_in + 3 * mc};
    PairBuf& pb = e->pairs[e->cur];
    const uint32_t S = e->n_slots;
    const uint64_t P = e->lim.max_pairs;
    const uint8_t* types = e->have_conn_type ? e->d_conn_type : nullptr;
    const unsigned blocks = blocks_for(9ull * n * 32, 256);
    {
        chd_status st0 = chd_epoch_tick(e, s, EP_BCAST);
        if (st0 != CHD_OK) return st0;
    }
    bcast_kernel<false><<<blocks, 256, 0, s>>>(e->g, bd, pb.off + S, P, pb, e->d_by_cell, e->d_conn, types, e->d_bc_cnt, nullptr, nullptr, 0,
                                               e->d_epoch + EP_BCAST);
    KCHECK(e);
    SCAN(e, exclusive_scan_1p<uint32_t, uint32_t>(e->d_bc_cnt, e->d_bc_off, 9ull * n, e->site_bcast, s));
    // (callable from any thread under the engine mutex: h_u32 is the mutex-protected scratch, as in chd_query_channel_ids)
    CU(e, cudaMemcpyAsync(e->h_u32, e->d_bc_off + 9ull * n, 4, cudaMemcpyDeviceToHost, s));
    CU(e, cudaStreamSynchronize(s));
    const uint32_t total = *e->h_u32;
    if (total > cap || (total && !out_slot)) {
        e->fail("chd_adjacent_broadcast: %u recipients > capacity %llu", total, (unsigned long long)cap);
        return CHD_ERR_CAPACITY;
    }
    if (!ensure_cap(e, &e->d_bc_out, &e->bc_out_cap, total, std::max<uint64_t>(1 << 16, (uint64_t)total + total / 2))) return CHD_ERR_CUDA;
    if (total) {
        bcast_kernel<true><<<blocks, 256, 0, s>>>(e->g, bd, pb.off + S, P, pb, e->d_by_cell, e->d_conn, types, nullptr, e->d_bc_off, e->d_bc_out,
                                                  e->bc_out_cap, nullptr);
        KCHECK(e);
        CU(e, cudaMemcpyAsync(out_slot, e->d_bc_out, 4ull * total, cudaMemcpyDefault, s));
    }
    bcast_msgoff_kernel<<<blocks_for((uint64_t)n + 1, 256), 256, 0, s>>>(e->d_bc_off, n, e->d_bc_msgoff);
    KCHECK(e);
    CU(e, cudaMemcpyAsync(out_off, e->d_bc_msgoff, 4ull * ((uint64_t)n + 1), cudaMemcpyDefault, s));
    CU(e, cudaStreamSynchronize(s));
    return CHD_OK;
}

uint32_t chd_get_adjacent_channels(const chd_grid_cfg* cfg, uint32_t channel_id, uint32_t* out8) {  // spatial.go:358-381
    if (!cfg || !out8 || cfg->grid_cols == 0) return 0;
    const uint32_t index = channel_id - cfg->channel_id_start;
    const int64_t gx = index % cfg->grid_cols, gy = index / cfg->grid_cols;
    uint32_t n = 0;
    for (int64_t y = gy - 1; y <= gy + 1; y++) {
        if (y < 0 || y >= (int64_t)cfg->grid_rows) continue;
        for (int64_t x = gx - 1; x <= gx + 1; x++) {
            if (x < 0 || x >= (int64_t)cfg->grid_cols) continue;
            if (x == gx && y == gy) continue;
            out8[n++] = (uint32_t)x + (uint32_t)y * cfg->grid_cols + cfg->channel_id_start;
        }
    }
    return n;
}

chd_status chd_get_regions(const chd_grid_cfg* cfg, double* min_x, double* min_z, double* max_x, double* max_z, uint32_t* channel_id,
                           uint32_t* server_index) {  // spatial.go:319-356
    if (!cfg || cfg->server_cols == 0 || cfg->server_rows == 0) return CHD_ERR_INVALID;
    uint32_t sgc = cfg->grid_cols / cfg->server_cols;
    if (cfg->grid_cols % cfg->server_cols) sgc++;
    uint32_t sgr = cfg->grid_rows / cfg->server_rows;
    if (cfg->grid_rows % cfg->server_rows) sgr++;
    for (uint32_t y = 0; y < cfg->grid_rows; y++)
        for (uint32_t x = 0; x < cfg->grid_cols; x++) {
            const uint32_t i = x + y * cfg->grid_cols;
            if (min_x) min_x[i] = cfg->world_offset_x + cfg->grid_width * (double)x;
            if (min_z) min_z[i] = cfg->world_offset_z + cfg->grid_height * (double)y;
            if (max_x) max_x[i] = cfg->world_offset_x + cfg->grid_width * (double)(x + 1);
            if (max_z) max_z[i] = cfg->world_offset_z + cfg->grid_height * (double)(y + 1);
            if (channel_id) channel_id[i] = cfg->channel_id_start + i;
            if (server_index) server_index[i] = (x / sgc) + (y / sgr) * cfg->server_cols;
        }
    return CHD_OK;
}
}  // extern "C"
