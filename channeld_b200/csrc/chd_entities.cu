// chd_entities.cu — entity positions, GetChannelId per entity, spatial-hash build (cell CSR).
#include "chd_engine.h"

#include "chd_build.cuh"
#include "chd_misc.cuh"

// assign: when set, the pass's histogram kernel also computes the keys from the positions (first pass of a single-GPU build)
struct FusedAssign {
    Positions pos;
    uint32_t* key;
    const uint32_t* prev;
    HandoverOut ho;
};

// One radix pass: digit (key >> shift) & mask of key[0, n) (n_ptr: the live length on the device), values val (nullptr: the
// index), block b of nblocks owns the slice [b * per_block, (b + 1) * per_block), histogram hist[digit][block].  Digits of up to
// 8 bits take 256 bins, wider ones 1024.
struct SortPass {
    const uint32_t *key, *val;
    uint32_t n;
    const uint32_t* n_ptr;
    uint32_t per_block, nblocks, shift, mask;
    uint32_t* hist;
};

// The pass's digit histogram (with assign: the cell assignment computes the keys and counts them in the same launch) and its
// exclusive scan, which leaves every block's base per digit
template <int BINS>
static chd_status count_digits(chd_engine* e, cudaStream_t s, const SortPass& p, const ScanSite& site, unsigned long long* bump,
                               const FusedAssign* assign) {
    if (assign)
        assign_hist_kernel<BINS><<<p.nblocks, BUILD_THREADS, 0, s>>>(e->g, assign->pos.x, assign->pos.z, p.n, assign->key, assign->prev, assign->ho, p.per_block,
                                                                     p.mask, p.hist, p.nblocks, bump);
    else
        radix_hist_kernel<BINS><<<p.nblocks, BUILD_THREADS, 0, s>>>(p.key, p.n, p.n_ptr, p.per_block, p.shift, p.mask, p.hist, p.nblocks, bump);
    KCHECK(e);
    SCAN(e, exclusive_scan_1p<uint32_t, uint32_t>(p.hist, p.hist, (uint64_t)BINS * p.nblocks, site, s));
    return CHD_OK;
}

// The pass's stable scatter from the scanned histogram.  Bandwidth-bound regime: each tile is reordered by digit in shared memory
// first (coalesced runs); small inputs are latency-bound and take the plain scatter (fewer barriers per tile).
template <int BINS>
static chd_status scatter_digits(chd_engine* e, cudaStream_t s, const SortPass& p, uint32_t* key_out, uint32_t* val_out, ScatterExtras ex) {
    if (p.n > (2u << 20))
        radix_scatter_sorted_kernel<BINS><<<p.nblocks, BUILD_THREADS, 0, s>>>(p.key, p.val, p.n, p.n_ptr, p.per_block, p.shift, p.mask, p.hist,
                                                                             p.nblocks, key_out, val_out, ex);
    else
        radix_scatter_kernel<BINS><<<p.nblocks, BUILD_THREADS, 0, s>>>(p.key, p.val, p.n, p.n_ptr, p.per_block, p.shift, p.mask, p.hist, p.nblocks,
                                                                      key_out, val_out, ex);
    KCHECK(e);
    return CHD_OK;
}

static chd_status count_pass(chd_engine* e, cudaStream_t s, const SortPass& p, const ScanSite& site, unsigned long long* bump,
                             const FusedAssign* assign) {
    return p.mask < 256 ? count_digits<256>(e, s, p, site, bump, assign) : count_digits<1024>(e, s, p, site, bump, assign);
}
static chd_status scatter_pass(chd_engine* e, cudaStream_t s, const SortPass& p, uint32_t* key_out, uint32_t* val_out, ScatterExtras ex = {}) {
    return p.mask < 256 ? scatter_digits<256>(e, s, p, key_out, val_out, ex) : scatter_digits<1024>(e, s, p, key_out, val_out, ex);
}

chd_status chd_cell_sort(chd_engine* e, cudaStream_t s, const CellSort& cs, uint32_t keys, const uint32_t* key, const uint32_t* val, uint32_t n,
                         const uint32_t* n_ptr, uint32_t* key_out, uint32_t* val_out, const ScatterExtras* csr, unsigned long long* bump,
                         const FusedAssign* assign, int part) {
    uint32_t bits = 1;
    while ((1u << bits) < keys) bits++;
    const uint32_t bits0 = bits <= 10 ? bits : (bits + 1) / 2;  // <= 2 passes of <= 10-bit digits
    // contiguous slice per block: a whole number of tiles, at least one
    const uint32_t slice = (uint32_t)(((uint64_t)n + cs.blocks - 1) / cs.blocks);
    const uint32_t per_block = std::max<uint32_t>(BUILD_TILE, (slice + BUILD_TILE - 1) / BUILD_TILE * BUILD_TILE);
    const uint32_t nblocks = cs.whole_grid ? cs.blocks : std::max(1u, (n + per_block - 1) / per_block);
    const SortPass p0{key, val, n, n_ptr, per_block, nblocks, 0, (1u << bits0) - 1u, cs.hist};
    chd_status st = CHD_OK;
    if (bits0 == bits) {  // one pass: digit == key, so block 0's scanned bases are the cell CSR offsets
        if (part != 2) {
            st = count_pass(e, s, p0, cs.site[0], bump, assign);
            if (st != CHD_OK) return st;
        }
        if (part != 1) return scatter_pass(e, s, p0, nullptr, val_out, part == 0 && csr ? *csr : ScatterExtras{});
        if (csr) {  // published before the scatter, so that the emit preparation can overlap it
            publish_cell_start_kernel<<<blocks_for((uint64_t)csr->cells + 2, 256), 256, 0, s>>>(cs.hist, nblocks, n, n_ptr, *csr);
            KCHECK(e);
        }
        return CHD_OK;
    }
    const SortPass p1{cs.tmp_key, cs.tmp_val, n, n_ptr, per_block, nblocks, bits0, (1u << (bits - bits0)) - 1u, cs.hist};
    st = count_pass(e, s, p0, cs.site[0], bump, assign);
    if (st == CHD_OK) st = scatter_pass(e, s, p0, cs.tmp_key, cs.tmp_val);
    if (st == CHD_OK) st = count_pass(e, s, p1, cs.site[1], nullptr, nullptr);
    if (st == CHD_OK) st = scatter_pass(e, s, p1, key_out, val_out);
    if (st != CHD_OK || !csr) return st;
    cell_bounds_kernel<<<blocks_for((uint64_t)n + 1, 256), 256, 0, s>>>(key_out, n, n_ptr, csr->cells, csr->cell_start, csr->n_in_world);
    KCHECK(e);
    return CHD_OK;
}

extern "C" {

/* ------------------------------------------------------------------ entities / build ---- */

chd_status chd_cell_of(chd_engine* e, const double* x, const double* z, uint32_t n, uint32_t* out) {
    return chd_cell_of_valid(e, x, z, n, out, nullptr);
}

chd_status chd_cell_of_valid(chd_engine* e, const double* x, const double* z, uint32_t n, uint32_t* out, uint8_t* out_valid) {
    if (!e || (n && (!x || !z || !out))) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_LOCK | ENTRY_DEVICE);
    // chunked through the tmp buffers (they are free outside chd_build)
    double *dx = nullptr, *dz = nullptr;
    uint32_t* dk = nullptr;
    uint8_t* dv = nullptr;
    const uint32_t chunk = 1u << 20;
    CU(e, cudaMallocAsync((void**)&dx, sizeof(double) * chunk, e->stream));
    CU(e, cudaMallocAsync((void**)&dz, sizeof(double) * chunk, e->stream));
    CU(e, cudaMallocAsync((void**)&dk, sizeof(uint32_t) * chunk, e->stream));
    if (out_valid) CU(e, cudaMallocAsync((void**)&dv, chunk, e->stream));
    HandoverOut ho{};
    for (uint32_t b = 0; b < n; b += chunk) {
        const uint32_t m = n - b < chunk ? n - b : chunk;
        CU(e, cudaMemcpyAsync(dx, x + b, sizeof(double) * m, cudaMemcpyDefault, e->stream));
        CU(e, cudaMemcpyAsync(dz, z + b, sizeof(double) * m, cudaMemcpyDefault, e->stream));
        assign_cells_kernel<<<blocks_for(m, 256), 256, 0, e->stream>>>(e->g, dx, dz, m, dk, nullptr, ho, nullptr);
        KCHECK(e);
        cell_key_to_id_kernel<<<blocks_for(m, 256), 256, 0, e->stream>>>(dk, m, e->g.cells, e->g.id_start, dv);
        KCHECK(e);
        CU(e, cudaMemcpyAsync(out + b, dk, sizeof(uint32_t) * m, cudaMemcpyDefault, e->stream));
        if (out_valid) CU(e, cudaMemcpyAsync(out_valid + b, dv, m, cudaMemcpyDefault, e->stream));
    }
    CU(e, cudaFreeAsync(dx, e->stream));
    CU(e, cudaFreeAsync(dz, e->stream));
    CU(e, cudaFreeAsync(dk, e->stream));
    if (dv) CU(e, cudaFreeAsync(dv, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

// float uploads (see widen_positions_kernel): the floats land in a staging buffer (or are read in place when they already live on
// the device) and are widened into the double buffers on the same stream, so everything downstream is unchanged.
static chd_status widen_upload(chd_engine* e, int which, const float* x, const float* z, uint32_t n, double* dx, double* dz, cudaStream_t s) {
    if (!n) return CHD_OK;
    const float *sx = x, *sz = z;
    if (!(chd_is_device_ptr(e, x) && chd_is_device_ptr(e, z))) {
        if (!e->d_pos_f32[which] && !dalloc(e, &e->d_pos_f32[which], 2ull * e->lim.max_entities + 8)) return CHD_ERR_CUDA;
        float* stage_x = e->d_pos_f32[which];
        float* stage_z = stage_x + (((size_t)e->lim.max_entities + 3) & ~(size_t)3);
        CU(e, cudaMemcpyAsync(stage_x, x, sizeof(float) * n, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(stage_z, z, sizeof(float) * n, cudaMemcpyDefault, s));
        sx = stage_x;
        sz = stage_z;
    } else if ((((uintptr_t)x) | ((uintptr_t)z)) & 15) {
        e->fail("float positions on the device must be 16-byte aligned");
        return CHD_ERR_INVALID;
    }
    widen_positions_kernel<<<blocks_for((n + 3) / 4, 256), 256, 0, s>>>(sx, sz, dx, dz, n);
    KCHECK(e);
    return CHD_OK;
}

void chd_entities_replaced(chd_engine* e, uint32_t n) {
    if (n != e->n_own) e->have_prev_key = false;
    e->n_own = n;
    e->n_halo = 0;
    e->halo_on_device = false;
    e->assigned = false;
    e->entities_dirty = true;
}

// argument checks of every position upload
static chd_status check_positions(chd_engine* e, const char* fn, const void* x, const void* z, uint32_t n) {
    if (!e || (n && (!x || !z))) return CHD_ERR_INVALID;
    if (chd_rule_not_table(e, fn) != CHD_OK) return CHD_ERR_STATE;
    if (n > e->lim.max_entities) {
        e->fail("%s: %u > max_entities %u", fn, n, e->lim.max_entities);
        return CHD_ERR_CAPACITY;
    }
    return CHD_OK;
}

// Every position upload, f64 or f32: into the front pair on the engine stream (set), or into the pair the next prefetch fills on
// up_stream (prefetch).  Device-resident doubles given to a set are read in place.
static chd_status upload_positions(chd_engine* e, const void* x, const void* z, uint32_t n, bool f32, bool prefetch) {
    int set = e->pf_pos.cur;
    chd_status st = prefetch ? chd_pf_begin(e, e->pf_pos, &set) : CHD_OK;
    if (st != CHD_OK) return st;
    cudaStream_t s = prefetch ? e->up_stream : e->stream;
    PosSet& p = e->pos[set];
    // the second pair of position buffers exists only for hosts that prefetch
    if (!p.z && !(dalloc(e, &p.x, e->lim.max_entities) && dalloc(e, &p.z, e->lim.max_entities))) return CHD_ERR_CUDA;
    const bool in_place = !f32 && !prefetch && n && chd_is_device_ptr(e, x) && chd_is_device_ptr(e, z);
    if (f32) {
        st = widen_upload(e, prefetch ? 1 : 0, (const float*)x, (const float*)z, n, p.x, p.z, s);
        if (st != CHD_OK) return st;
    } else if (!in_place) {
        CU(e, cudaMemcpyAsync(p.x, x, sizeof(double) * n, cudaMemcpyDefault, s));
        CU(e, cudaMemcpyAsync(p.z, z, sizeof(double) * n, cudaMemcpyDefault, s));
    }
    if (prefetch) {
        p.n = n;
        return chd_pf_end(e, e->pf_pos);
    }
    e->in_place = in_place ? Positions{(const double*)x, (const double*)z} : Positions{};  // device-resident producer: read in place
    chd_entities_replaced(e, n);
    return CHD_OK;
}

chd_status chd_set_entities(chd_engine* e, const double* x, const double* z, uint32_t n) {
    const chd_status st = check_positions(e, "chd_set_entities", x, z, n);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return upload_positions(e, x, z, n, false, false);
}
chd_status chd_prefetch_entities(chd_engine* e, const double* x, const double* z, uint32_t n) {
    const chd_status st = check_positions(e, "chd_prefetch_entities", x, z, n);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return upload_positions(e, x, z, n, false, true);
}
chd_status chd_set_entities_f32(chd_engine* e, const float* x, const float* z, uint32_t n) {
    const chd_status st = check_positions(e, "chd_set_entities_f32", x, z, n);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return upload_positions(e, x, z, n, true, false);
}
chd_status chd_prefetch_entities_f32(chd_engine* e, const float* x, const float* z, uint32_t n) {
    const chd_status st = check_positions(e, "chd_prefetch_entities_f32", x, z, n);
    if (st != CHD_OK) return st;
    CHD_ENTER(e, ENTRY_DEVICE);
    return upload_positions(e, x, z, n, true, true);
}

chd_status chd_entity_buffers(chd_engine* e, double** x, double** z, uint32_t* n) {
    if (!e) return CHD_ERR_INVALID;
    if (chd_rule_not_table(e, "chd_entity_buffers") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, 0);
    if (x) *x = chd_pos_front(e).x;
    if (z) *z = chd_pos_front(e).z;
    if (n) *n = e->n_own;
    e->in_place = {};
    e->assigned = false;  // the caller may write positions
    e->entities_dirty = true;
    return CHD_OK;
}

chd_status chd_set_entity_count(chd_engine* e, uint32_t n) {
    if (!e || n > e->lim.max_entities) return CHD_ERR_INVALID;
    if (chd_rule_not_table(e, "chd_set_entity_count") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, 0);
    chd_entities_replaced(e, n);
    return CHD_OK;
}

chd_status chd_set_entity_ids(chd_engine* e, const uint32_t* gid, uint32_t n) {
    if (!e || n > e->lim.max_entities) return CHD_ERR_INVALID;
    if (chd_rule_not_table(e, "chd_set_entity_ids") != CHD_OK) return CHD_ERR_STATE;
    CHD_ENTER(e, ENTRY_DEVICE);
    e->delta_blocked = true;  // global ids: the multi-GPU flow (index-mode visible deltas are single-GPU only)
    if (!gid) {
        e->have_gid = false;
        return CHD_OK;
    }
    CU(e, cudaMemcpyAsync(e->d_gid, gid, sizeof(uint32_t) * n, cudaMemcpyDefault, e->stream));
    e->have_gid = true;
    e->entities_dirty = true;
    return CHD_OK;
}

chd_status chd_assign_cells(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_FETCH_GUARD);
    const bool was_assigned = e->assigned;
    chd_status st = chd_assign_cells_impl(e, e->stream);
    if (st == CHD_OK && !was_assigned) st = chd_note_pos_read(e, e->stream);
    return st;
}

uint32_t* chd_assign_host(chd_engine* e) {
    uint32_t* prev = nullptr;
    if (e->have_prev_key) {
        std::swap(e->d_key, e->d_prev_key);
        prev = e->d_prev_key;
    }
    if (e->n_own) e->have_prev_key = true;
    e->n_halo = 0;
    e->assigned = true;
    e->tbl.ho_raw = true;  // (entity-table mode: the handover list now names slots until chd_table_after_build)
    return prev;
}

// chd_assign_host, the handover output and its counter zeroed on `s`
static chd_status assign_prepare(chd_engine* e, cudaStream_t s, uint32_t** prev_out, HandoverOut* ho) {
    *prev_out = chd_assign_host(e);
    *ho = HandoverOut{e->d_ho_entity, e->d_ho_src, e->d_ho_dst, &e->d_ctr->n_handover, e->ho_cap};
    CU(e, cudaMemsetAsync(&e->d_ctr->n_handover, 0, 4, s));
    return CHD_OK;
}

chd_status chd_assign_cells_impl(chd_engine* e, cudaStream_t s) {
    if (e->assigned) return CHD_OK;
    uint32_t* prev = nullptr;
    HandoverOut ho{};
    chd_status st = assign_prepare(e, s, &prev, &ho);
    if (st != CHD_OK) return st;
    if (e->n_own) {
        const Positions p = chd_positions(e);
        assign_cells_kernel<<<blocks_for(e->n_own, 256), 256, 0, s>>>(e->g, p.x, p.z, e->n_own, e->d_key, prev, ho, e->assign_bump);
        KCHECK(e);
        e->assign_bump = nullptr;  // consumed
    }
    return CHD_OK;
}

// The cell CSR into copy-input set `out`.  part: 0 = the whole build; single-pass builds only: 1 = cell assignment + histogram +
// scan + CSR offsets, 2 = scatter.  The cell CSR offsets are final after part 1.
static chd_status build_enqueue(chd_engine* e, cudaStream_t s, const CopySet& out, bool with_assign, int part = 0) {
    chd_status st;
    FusedAssign fa{};
    const FusedAssign* fap = nullptr;
    if (with_assign) {
        if (!e->assigned && e->n_own && !e->halo_on_device) {
            // single-GPU build: GetChannelId per entity is fused into the first pass's histogram kernel
            uint32_t* prev = nullptr;
            HandoverOut ho{};
            st = assign_prepare(e, s, &prev, &ho);
            if (st != CHD_OK) return st;
            fa = FusedAssign{chd_positions(e), e->d_key, prev, ho};
            fap = &fa;
        } else {
            st = chd_assign_cells_impl(e, s);
            if (st != CHD_OK) return st;
        }
    }
    // multi-GPU: the halo count stays on the device (d_n_build = own + kept halo records); launches are sized for
    // the entity capacity and blocks beyond the live length idle.
    const uint32_t* n_ptr = e->halo_on_device ? e->d_n_build : nullptr;
    const uint32_t n = e->halo_on_device ? e->lim.max_entities : e->n_own + e->n_halo;
    const ScatterExtras csr{out.cell_start, e->g.cells, &e->d_ctr->n_entities_in_world};
    // keys are in [0, C]: C marks an out-of-world entity
    return chd_cell_sort(e, s, e->ent_sort, e->g.cells + 1, e->d_key, e->have_gid ? e->d_gid : nullptr, n, n_ptr, e->d_sorted_key, out.sorted_ent,
                         &csr, e->d_epoch + EP_BUILD, fap, part);
}

chd_status chd_build(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD);
    return chd_build_on(e, e->stream);
}

chd_status chd_build_on(chd_engine* e, cudaStream_t s) {
    StageTimer timer(e, s, CHD_STAGE_BUILD);
    // The cell CSR goes to the copy-input set the last copy kernel did not read, once every copy kernel that read it has finished.
    // X-slabs keep one set: chd_tick_sharded joins its copy kernel inside the tick, so nothing of the next tick runs beside it.
    int set = e->pf_copy.cur;
    chd_status st = e->slab ? CHD_OK : chd_pf_begin(e, e->pf_copy, &set, s);
    if (st != CHD_OK) return st;
    const CopySet& out = e->copy_set[set];
    st = chd_epoch_tick(e, s, EP_BUILD);
    if (st != CHD_OK) return st;
    bool counts_recorded = false;
    if (!e->assigned && !e->halo_on_device) {
        // single-GPU flow: assign + sort as one replayable graph.  The key buffers swap every assignment (handover detection
        // compares against the previous keys); the graph bakes in the sizes, the buffer the new keys go to and the positions.
        const uint64_t key = stage_key(0x6275696c64ull, e->n_own, e->have_gid, e->have_prev_key, e->have_prev_key ? e->d_prev_key : e->d_key,
                                       chd_positions(e).x, chd_positions(e).z, set);
        // single-pass builds (<= 1023 cells) run as two replayable halves with an event in between: the cell CSR offsets are
        // final after the first (assignment + histogram + scan), so the emit preparation overlaps the scatter
        const bool split = e->g.cells + 1 <= BUILD_MAX_BINS && e->n_own > 0;
        st = run_stage(e, s, e->g_build, key, [&]() { return build_enqueue(e, s, out, true, split ? 1 : 0); });
        if (st == CHD_OK && !e->assigned) chd_assign_host(e);  // replayed graph
        if (st == CHD_OK && split) {
            CU(e, cudaEventRecord(e->ev_counts, s));
            counts_recorded = true;
            st = run_stage(e, s, e->g_build_b, stage_key(key, 0x62), [&]() { return build_enqueue(e, s, out, false, 2); });
        }
        if (st == CHD_OK) st = chd_note_pos_read(e, s);
    } else if (e->assigned && e->halo_on_device) {
        // multi-GPU flow: cells were assigned by chd_export_border and the halo appended on the device; the sort over
        // own + halo entities is sized by capacity (device-side length) and therefore replayable as well.
        const uint64_t key = stage_key(0x736f7274ull, e->lim.max_entities, e->have_gid, e->d_key, set);
        st = run_stage(e, s, e->g_build, key, [&]() { return build_enqueue(e, s, out, false); });
    } else {
        const bool with_assign = !e->assigned;
        st = build_enqueue(e, s, out, with_assign);
        if (st == CHD_OK && with_assign) st = chd_note_pos_read(e, s);
    }
    if (st != CHD_OK) return st;
    st = chd_table_after_build(e, s, out);  // (entity-table mode only)
    if (st != CHD_OK) return st;
    if (!counts_recorded) CU(e, cudaEventRecord(e->ev_counts, s));  // (cell counts final = build done)
    if (!e->slab) {
        st = chd_pf_end(e, e->pf_copy, s);
        if (st != CHD_OK) return st;
        chd_pf_adopt(e->pf_copy);
    }
    e->n_sorted = e->n_own + e->n_halo;
    e->sorted_dev_n = e->halo_on_device;
    e->built = true;
    e->entities_dirty = false;
    return CHD_OK;
}
}  // extern "C"
