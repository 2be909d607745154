// chd_engine.cu — engine object: create / destroy, streams, memory, look-back scan sites, instrumentation.
#include "chd_engine.h"

static thread_local std::string g_create_error;

// epochs start at 1 so that the zero-initialised descriptors (epoch 0) read as stale on first use
bool chd_init_epochs(chd_engine* e) {
    unsigned long long ones[EP_COUNT];
    for (unsigned long long& v : ones) v = 1;
    return cudaMemcpy(e->d_epoch, ones, sizeof ones, cudaMemcpyHostToDevice) == cudaSuccess;
}

bool chd_make_site(chd_engine* e, ScanSite& site, uint64_t n_max, int stage) {
    site.tiles = n_max == 0 ? 1 : (n_max + SCAN_TILE - 1) / SCAN_TILE;
    site.epoch = e->d_epoch + stage;
    site.error = e->d_ctr ? &e->d_ctr->overflow : nullptr;  // (sites made before d_ctr exists are patched in chd_create)
    site.stage = stage;
    if (std::find(e->sites.begin(), e->sites.end(), &site) == e->sites.end()) e->sites.push_back(&site);
    if (!dalloc(e, &site.desc, site.tiles)) return false;
    return cudaMemset(site.desc, 0, site.tiles * 8) == cudaSuccess;
}

// Zero-copy inputs: a pointer into this device's memory is consumed in place (no staging copy); the caller keeps it valid
// and unmodified until the work that reads it has finished (chd_summary / chd_sync / any chd_get_*).
bool chd_is_device_ptr(const chd_engine* e, const void* p) {
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice && a.device == e->device;
}

chd_status chd_epoch_tick(chd_engine* e, cudaStream_t s, int stage) {
    if ((++e->stage_execs[stage] & ((1ull << 20) - 1)) != 0) return CHD_OK;
    for (ScanSite* site : e->sites)
        if (site->stage == stage && site->desc) CU(e, cudaMemsetAsync(site->desc, 0, site->tiles * 8, s));
    return CHD_OK;
}

void chd_dfree(chd_engine* e, void* p) {
    if (!p) return;
    for (size_t i = 0; i < e->allocs.size(); i++)
        if (e->allocs[i] == p) {
            e->allocs.erase(e->allocs.begin() + (long)i);
            break;
        }
    cudaFree(p);
}

static bool pf_events(chd_engine* e, Prefetch& p) {
    if (p.ev_read[1]) return true;  // (made last)
    return chd_make_event(e, &p.ev_upload) && chd_make_event(e, &p.ev_read[0]) && chd_make_event(e, &p.ev_read[1]);
}

chd_status chd_pf_begin(chd_engine* e, Prefetch& p, int* set, cudaStream_t s) {
    if (!s && !e->up_stream && !chd_make_stream(e, &e->up_stream)) return CHD_ERR_CUDA;
    if (!pf_events(e, p)) return CHD_ERR_CUDA;
    if (chd_pf_after_read(e, p, p.next, s ? s : e->up_stream) != CHD_OK) return CHD_ERR_CUDA;
    *set = p.next;
    p.staged = -1;  // a staged upload is in this set: an upload that fails part way leaves nothing staged
    return CHD_OK;
}

chd_status chd_pf_end(chd_engine* e, Prefetch& p, cudaStream_t s) {
    CU(e, cudaEventRecord(p.ev_upload, s ? s : e->up_stream));
    p.staged = p.next;
    return CHD_OK;
}

bool chd_pf_adopt(Prefetch& p) {
    if (p.staged < 0) return false;
    p.cur = p.staged;
    p.next = p.staged ^ 1;
    p.staged = -1;
    p.wait = true;
    return true;
}

chd_status chd_pf_wait(chd_engine* e, Prefetch& p, cudaStream_t s) {
    if (!p.wait) return CHD_OK;
    CU(e, cudaStreamWaitEvent(s, p.ev_upload, 0));
    p.wait = false;
    return CHD_OK;
}

chd_status chd_pf_note_read(chd_engine* e, Prefetch& p, int set, cudaStream_t s) {
    if (set < 0) return CHD_OK;
    if (!pf_events(e, p)) return CHD_ERR_CUDA;
    CU(e, cudaEventRecord(p.ev_read[set], s));
    p.read_recorded[set] = true;
    return CHD_OK;
}

chd_status chd_pf_after_read(chd_engine* e, const Prefetch& p, int set, cudaStream_t s) {
    if (p.read_recorded[set]) CU(e, cudaStreamWaitEvent(s, p.ev_read[set], 0));
    return CHD_OK;
}

cudaError_t chd_copy_wait(chd_engine* e) {
    if (e->copy_pending < 0) return cudaSuccess;
    const cudaError_t r = cudaStreamWaitEvent(e->stream, e->pf_copy.ev_read[e->copy_pending], 0);
    if (r == cudaSuccess) e->copy_pending = -1;
    return r;
}

chd_status chd_enter(chd_engine* e, unsigned needs, std::unique_lock<std::recursive_mutex>& lock) {
    if (needs & ENTRY_LOCK) lock = std::unique_lock<std::recursive_mutex>(e->mu);
    if (!(needs & (ENTRY_DEVICE | ENTRY_COPY_WAIT | ENTRY_FETCH_GUARD))) return CHD_OK;
    CU(e, cudaSetDevice(e->device));
    if (needs & ENTRY_COPY_WAIT) CU(e, chd_copy_wait(e));
    return needs & ENTRY_FETCH_GUARD ? chd_fetch_guard(e, e->stream) : CHD_OK;
}

chd_status chd_read_u32(chd_engine* e, const uint32_t* d, uint32_t* v) {
    CU(e, cudaMemcpyAsync(e->h_get, d, 4, cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    *v = *e->h_get;
    return CHD_OK;
}

extern "C" {

uint32_t chd_abi_version(void) { return CHD_ABI_VERSION; }

uint32_t chd_damping_interval_ms(uint32_t dist, uint32_t default_ms) { return damping_interval_ms(dist, default_ms); }

void chd_default_limits(const chd_grid_cfg* cfg, uint32_t n_entities, uint32_t n_subscribers, chd_limits* lim) {
    memset(lim, 0, sizeof *lim);
    const uint64_t cells = (uint64_t)cfg->grid_cols * cfg->grid_rows;
    lim->max_entities = n_entities ? n_entities : 1;
    lim->max_subscribers = n_subscribers ? n_subscribers : 1;
    lim->max_queries = lim->max_subscribers;
    lim->max_spots = 1024;
    lim->max_pairs = (uint64_t)lim->max_subscribers * 16 + 1024;
    lim->max_window_cells = (uint64_t)lim->max_queries * 32 + 65536;
    const double per_cell = (double)n_entities / (double)(cells ? cells : 1);
    double v = (double)n_subscribers * 1.6 * per_cell * 1.5 + 1048576.0;
    if (v > 3.0e9) v = 3.0e9;
    lim->max_visible = (uint64_t)v;
    lim->max_ring_entries = (uint32_t)(cells * 64 < 1048576 ? 1048576 : (cells * 64 > 0x7fffffffull ? 0x7fffffffull : cells * 64));
    lim->max_due = (uint32_t)(lim->max_pairs * 2 > 0x7fffffffull ? 0x7fffffffull : lim->max_pairs * 2);
    lim->default_fanout_interval_ms = 20;  // GLOBAL defaults, settings.go:97-103
    lim->default_fanout_delay_ms = 0;
}

const char* chd_last_error(const chd_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

// NUMA node the GPU hangs off (sysfs), -1 if unknown: a host that runs its tick driver on that node's cores gets node-local
// pinned staging memory by first touch (measured: 37 GB/s -> > 50 GB/s H2D on the bench box when the staging memory is local)
int chd_device_numa_node(int device) {
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    for (char* p = bus; *p; p++)
        if (*p >= 'A' && *p <= 'Z') *p = (char)(*p - 'A' + 'a');
    char path[160];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

void* chd_alloc_pinned(uint64_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
void chd_free_pinned(void* p) {
    if (p) cudaFreeHost(p);
}

void chd_destroy(chd_engine* e) {
    if (!e) return;
    // device and copy wait without CHD_ENTER: the engine is released whatever fails (a void call has no status to return)
    cudaSetDevice(e->device);
    if (e->stream) {
        chd_copy_wait(e);
        cudaStreamSynchronize(e->stream);
    }
    chd_comm_destroy(e);
    for (cudaStream_t s : e->streams) cudaStreamSynchronize(s);
    for (void* p : e->allocs) cudaFree(p);
    for (cudaEvent_t ev : e->events) cudaEventDestroy(ev);
    for (cudaStream_t s : e->streams) cudaStreamDestroy(s);
    if (e->ev) {
        for (size_t i = 0; i < (size_t)CHD_STAGE_COUNT * chd_engine::EV_RING * 2; i++)
            if (e->ev[i]) cudaEventDestroy(e->ev[i]);
        delete[] e->ev;
    }
    if (e->h_ctr) cudaFreeHost(e->h_ctr);
    if (e->h_u32) cudaFreeHost(e->h_u32);
    if (e->h_get) cudaFreeHost(e->h_get);
    for (uint8_t* h : e->tbl.h_stage)
        if (h) cudaFreeHost(h);
    if (e->own_stream && e->stream) cudaStreamDestroy(e->stream);
    delete e;  // on e->device: the graph slots release their executables
}

static bool alloc_pairbuf(chd_engine* e, PairBuf& pb) {
    const uint64_t P = e->lim.max_pairs;
    return dalloc(e, &pb.off, (uint64_t)e->lim.max_subscribers + 1) && dalloc(e, &pb.sub, P) && dalloc(e, &pb.cell, P) &&
           dalloc(e, &pb.dist, P) && dalloc(e, &pb.interval, P) && dalloc(e, &pb.flags, P) && dalloc(e, &pb.last, P) &&
           dalloc(e, &pb.last_index, P);
}

// a sort by cell on `blocks` blocks, its scans in `stage`.  The caller allocates the temporaries in their place in chd_create's
// order: where the large buffers land moves the emit kernel's time (moving the entity sort's here cost 1.5 % of bench.py's
// benchmark config on an H100 80GB HBM3 at 700 W)
static bool alloc_cell_sort(chd_engine* e, CellSort& cs, uint32_t blocks, bool whole_grid, int stage) {
    const uint64_t bins = (uint64_t)BUILD_MAX_BINS * blocks;
    cs.blocks = blocks;
    cs.whole_grid = whole_grid;
    return dalloc(e, &cs.hist, bins + 2) && chd_make_site(e, cs.site[0], bins + 1, stage) && chd_make_site(e, cs.site[1], bins + 1, stage);
}

chd_status chd_create(const chd_grid_cfg* cfg, const chd_limits* lim_in, int device, chd_engine** out) {
    if (!cfg || !out) {
        g_create_error = "null argument";
        return CHD_ERR_INVALID;
    }
    *out = nullptr;
    // LoadConfig validation (spatial.go:146-154); ServerInterestBorderSize == 0 tolerated (see header)
    if (!(cfg->grid_width > 0) || !(cfg->grid_height > 0)) {
        g_create_error = "GridWidth and GridHeight should be positive";
        return CHD_ERR_INVALID;
    }
    if (cfg->grid_cols == 0 || cfg->grid_rows == 0) {
        g_create_error = "GridCols and GridRows should be positive";
        return CHD_ERR_INVALID;
    }
    if (cfg->server_cols == 0 || cfg->server_rows == 0) {
        g_create_error = "ServerCols and ServerRows should be positive";
        return CHD_ERR_INVALID;
    }
    const uint64_t cells64 = (uint64_t)cfg->grid_cols * cfg->grid_rows;
    if (cells64 >= (1ull << 20)) {  // spatial id space is [0x10000, 0x80000) (settings.go:94-95): < 2^19 cells
        g_create_error = "too many cells (GridCols*GridRows must be < 2^20)";
        return CHD_ERR_INVALID;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        g_create_error = "no CUDA device: this engine has no CPU fallback";
        return CHD_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) {
        g_create_error = "bad device ordinal";
        return CHD_ERR_INVALID;
    }
    chd_engine* e = new (std::nothrow) chd_engine();
    if (!e) return CHD_ERR_INVALID;
    e->cfg = *cfg;
    if (lim_in)
        e->lim = *lim_in;
    else
        chd_default_limits(cfg, 1u << 20, 1u << 17, &e->lim);
    chd_limits& L = e->lim;
    if (!L.max_entities) L.max_entities = 1;
    if (!L.max_subscribers) L.max_subscribers = 1;
    if (!L.max_queries) L.max_queries = L.max_subscribers;
    if (!L.max_pairs) L.max_pairs = 1024;
    if (!L.max_window_cells) L.max_window_cells = 65536;
    if (!L.max_visible) L.max_visible = 1u << 20;
    if (!L.max_ring_entries) L.max_ring_entries = 1u << 16;
    if (!L.max_due) L.max_due = 1u << 16;
    if (L.max_pairs >= 0xFFFFFFF0ull || L.max_window_cells >= (1ull << 40) || L.max_entities >= (1u << 30)) {
        g_create_error = "limits too large (pairs are indexed with 32 bits)";
        delete e;
        return CHD_ERR_INVALID;
    }
    e->device = device;
#define CCU(call)                                                                       \
    do {                                                                                \
        cudaError_t _r = (call);                                                        \
        if (_r != cudaSuccess) {                                                        \
            g_create_error = std::string(#call " failed: ") + cudaGetErrorString(_r);   \
            chd_destroy(e);                                                             \
            return CHD_ERR_CUDA;                                                        \
        }                                                                               \
    } while (0)
    CCU(cudaSetDevice(device));
    CCU(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    e->own_stream = true;
    CCU(cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, device));
    CCU(cudaDeviceGetAttribute(&e->l2_bytes, cudaDevAttrL2CacheSize, device));

    GridDev& g = e->g;
    g.off_x = cfg->world_offset_x; g.off_z = cfg->world_offset_z; g.w = cfg->grid_width; g.h = cfg->grid_height;
    g.grid_size = std::sqrt(g.w * g.w + g.h * g.h);                  // spatial.go:134-139
    g.world_x_hi = g.off_x + g.w * (double)cfg->grid_cols;           // spatial.go:126-132,287
    g.world_z_hi = g.off_z + g.h * (double)cfg->grid_rows;
    g.fcols = (double)cfg->grid_cols; g.frows = (double)cfg->grid_rows;
    g.cols = cfg->grid_cols; g.rows = cfg->grid_rows; g.cells = (uint32_t)cells64; g.id_start = cfg->channel_id_start;
    g.col_lo = 0; g.col_hi = g.cols; g.halo = 0;
    g.default_interval_ms = L.default_fanout_interval_ms; g.default_delay_ms = L.default_fanout_delay_ms;

    const uint64_t N = L.max_entities, S = L.max_subscribers, Q = L.max_queries, P = L.max_pairs, C = g.cells;
    e->ho_cap = L.max_entities;
    e->max_tiles = (L.max_visible + EMIT_WARP_TILE - 1) / EMIT_WARP_TILE + 1;  // (the smaller of the two tile sizes)
    // the aux stream carries short latency-bound kernels that should slot in ahead of the long emit kernel
    bool ok = chd_make_stream(e, &e->aux_stream) && chd_make_stream(e, &e->dl_stream) && chd_make_stream(e, &e->dl_stream_b) &&
              chd_make_stream(e, &e->prep_stream) && chd_make_stream(e, &e->build_stream) && chd_make_stream(e, &e->copy_stream, true);
    for (cudaEvent_t* ev : {&e->ev_fork, &e->ev_join, &e->ev_interest, &e->ev_pairs, &e->ev_prep_done, &e->ev_build_done, &e->ev_counts})
        ok = ok && chd_make_event(e, ev);
    e->pf_pos.cur = 0;  // the pair allocated here is the front one; the first prefetch fills the other
    e->pf_pos.next = 1;
    ok = ok && dalloc(e, &e->pos[0].x, N) && dalloc(e, &e->pos[0].z, N) && dalloc(e, &e->d_gid, N) && dalloc(e, &e->d_key, N) &&
         dalloc(e, &e->d_prev_key, N) && dalloc(e, &e->ent_sort.tmp_key, N) && dalloc(e, &e->ent_sort.tmp_val, N) &&
         dalloc(e, &e->d_sorted_key, N) &&
         // padded: an emit chunk that starts m != 0 entries into an aligned 16-byte chunk also loads the next aligned chunk,
         // which near the end of the array lies past N (chd_emit.cuh)
         dalloc(e, &e->copy_set[0].sorted_ent, ((N + 3) / 4) * 4 + 8) && dalloc(e, &e->copy_set[1].sorted_ent, ((N + 3) / 4) * 4 + 8) &&
         dalloc(e, &e->copy_set[0].cell_start, C + 2) && dalloc(e, &e->copy_set[1].cell_start, C + 2) &&
         dalloc(e, &e->d_epoch, EP_COUNT) && chd_init_epochs(e) &&
         alloc_cell_sort(e, e->ent_sort, (uint32_t)e->sm_count * 4, false, EP_BUILD) &&
         chd_make_site(e, e->site_qoff, Q + 1, EP_QUERY) && chd_make_site(e, e->site_slot, S + 1, EP_QUERY) &&
         chd_make_site(e, e->site_voff, P + 1, EP_EMIT) &&
         chd_make_site(e, e->site_border, N + 1, EP_BORDER) &&
         dalloc(e, &e->d_ho_entity, N) && dalloc(e, &e->d_ho_src, N) && dalloc(e, &e->d_ho_dst, N) &&
         dalloc(e, &e->d_bflag, N + 1) && dalloc(e, &e->d_boff, N + 2);
    ok = ok && dalloc(e, &e->d_conn, S) && dalloc(e, &e->d_slot_ctl, S) && dalloc(e, &e->d_slot_src, S) && dalloc(e, &e->d_lc_slot, S) &&
         dalloc(e, &e->d_lc_aux, S) && alloc_pairbuf(e, e->pairs[0]) && alloc_pairbuf(e, e->pairs[1]);
    ok = ok && alloc_qstage(e, e->dq);
    ok = ok && dalloc(e, &e->d_bbox, Q) && dalloc(e, &e->d_win_off, Q + 1) && dalloc(e, &e->d_qstatus, Q) && dalloc(e, &e->d_win_cursor, 1) &&
         dalloc(e, &e->d_noff, S + 2) &&
         dalloc(e, &e->d_window, L.max_window_cells) && dalloc(e, &e->d_side_cell, (uint64_t)L.max_spots) &&
         dalloc(e, &e->d_side_dist, (uint64_t)L.max_spots) && dalloc(e, &e->d_side_cnt, Q) && dalloc(e, &e->d_status, Q) &&
         dalloc(e, &e->d_qcount, Q) && dalloc(e, &e->d_qoff, Q + 1) && dalloc(e, &e->d_qout_id, P) && dalloc(e, &e->d_qout_dist, P) &&
         dalloc(e, &e->d_slot_query, S);
    ok = ok && dalloc(e, &e->d_new_off, (Q > P ? Q : P) + 2) && dalloc(e, &e->d_new_sub, P) && dalloc(e, &e->d_new_ch, P) && dalloc(e, &e->d_gone_sub, P) &&
         dalloc(e, &e->d_gone_ch, P);
    ok = ok && dalloc(e, &e->d_pair_ch, P) && dalloc(e, &e->d_vcnt, P) && dalloc(e, &e->d_vis_off, S + 1) && dalloc(e, &e->d_vis, L.max_visible);
    for (CopySet& c : e->copy_set)
        ok = ok && dalloc(e, &c.voff, P + 1) && dalloc(e, &c.first_pair, e->max_tiles + 8) && dalloc(e, &c.tile_desc, (L.max_visible + EMIT_TILE - 1) / EMIT_TILE + 8) &&
             dalloc(e, &c.general_tiles, (L.max_visible + EMIT_TILE - 1) / EMIT_TILE + 8) && dalloc(e, &c.n_general, 4) && dalloc(e, &c.n_visible, 1);
    ok = ok && dalloc(e, &e->d_cell_max_interval, C) && dalloc(e, &e->d_cell_start_ns, C) && chd_rings_create(e) == CHD_OK && dalloc(e, &e->d_by_cell, P) &&
         alloc_cell_sort(e, e->pair_sort, (uint32_t)std::min<uint64_t>(4096, (P + BUILD_TILE - 1) / BUILD_TILE), true, EP_QUERY) &&
         dalloc(e, &e->pair_sort.tmp_key, P) && dalloc(e, &e->pair_sort.tmp_val, P) &&
         dalloc(e, &e->d_due, (uint64_t)L.max_due) && dalloc(e, &e->d_due_key, (uint64_t)L.max_due) && dalloc(e, &e->d_ctr, 1) && dalloc(e, &e->d_time, 2) &&
         dalloc(e, &e->d_n_build, 1);
    if (!ok) {
        g_create_error = e->err;
        chd_destroy(e);
        return CHD_ERR_CUDA;
    }
    for (ScanSite* site : e->sites)
        site->error = &e->d_ctr->overflow;
    CCU(cudaHostAlloc((void**)&e->h_ctr, sizeof(Counters), cudaHostAllocDefault));
    CCU(cudaHostAlloc((void**)&e->h_u32, 64, cudaHostAllocDefault));
    CCU(cudaHostAlloc((void**)&e->h_get, 64, cudaHostAllocDefault));
    CCU(cudaMemsetAsync(e->d_ctr, 0, sizeof(Counters), e->stream));
    CCU(cudaMemsetAsync(e->d_win_cursor, 0, 8, e->stream));
    for (CopySet& c : e->copy_set) {
        CCU(cudaMemsetAsync(c.n_general, 0, 16, e->stream));
        CCU(cudaMemsetAsync(c.n_visible, 0, 8, e->stream));
        CCU(cudaMemsetAsync(c.cell_start, 0, (C + 2) * 4, e->stream));
    }
    e->pf_copy.cur = 0;  // a build fills set 1 first
    e->pf_copy.next = 1;
    CCU(cudaMemsetAsync(e->d_slot_ctl, 0, S, e->stream));
    CCU(cudaMemsetAsync(e->d_cell_max_interval, 0, C * 4, e->stream));
    CCU(cudaMemsetAsync(e->d_cell_start_ns, 0, C * 8, e->stream));
    CCU(cudaMemsetAsync(e->d_conn, 0, S * 4, e->stream));
    CCU(cudaMemsetAsync(e->d_time, 0, 16, e->stream));
    CCU(cudaMemsetAsync(e->pairs[0].off, 0, (S + 1) * 4, e->stream));
    CCU(cudaMemsetAsync(e->pairs[1].off, 0, (S + 1) * 4, e->stream));
    CCU(cudaMemsetAsync(e->d_vis_off, 0, (S + 1) * 8, e->stream));
    CCU(cudaStreamSynchronize(e->stream));
#undef CCU
    *out = e;
    return CHD_OK;
}

chd_status chd_set_stream(chd_engine* e, void* cuda_stream) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_DEVICE);
    CU(e, cudaStreamSynchronize(e->stream));
    if (e->own_stream) {
        cudaStreamDestroy(e->stream);
        e->own_stream = false;
    }
    e->stream = (cudaStream_t)cuda_stream;
    return CHD_OK;
}

chd_status chd_sync(chd_engine* e) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaStreamSynchronize(e->stream));
    return CHD_OK;
}

/* ------------------------------------------------------------------ instrumentation ---- */

uint64_t chd_launch_count(const chd_engine* e) { return e ? e->n_launch : 0; }

chd_status chd_enable_graphs(chd_engine* e, int on) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, 0);
    e->use_graphs = on != 0;
    return CHD_OK;
}

uint64_t chd_graph_launch_count(const chd_engine* e) { return e ? e->graph_launches : 0; }

chd_status chd_profile_enable(chd_engine* e, int on) {
    if (!e) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    if (on && !e->ev) {
        const size_t n = (size_t)CHD_STAGE_COUNT * chd_engine::EV_RING * 2;
        e->ev = new cudaEvent_t[n]();
        for (size_t i = 0; i < n; i++) CU(e, cudaEventCreate(&e->ev[i]));
    }
    CU(e, cudaStreamSynchronize(e->stream));
    for (int s = 0; s < CHD_STAGE_COUNT; s++) e->stage_n[s] = 0;
    e->profiling = on == 2 ? 2 : (on != 0 ? 1 : 0);
    return CHD_OK;
}

chd_status chd_profile_timeline(chd_engine* e, int stage, double* start_ms, double* stop_ms) {
    if (!e || stage < 0 || stage >= CHD_STAGE_COUNT || !start_ms || !stop_ms || !e->ev) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaStreamSynchronize(e->stream));
    CU(e, cudaStreamSynchronize(e->aux_stream));
    if (!e->stage_n[CHD_STAGE_TICK] || !e->stage_n[stage]) return CHD_ERR_STATE;
    cudaEvent_t t0 = e->evt(CHD_STAGE_TICK, e->stage_n[CHD_STAGE_TICK] - 1, 0);
    float a = 0, b = 0;
    CU(e, cudaEventElapsedTime(&a, t0, e->evt(stage, e->stage_n[stage] - 1, 0)));
    CU(e, cudaEventElapsedTime(&b, t0, e->evt(stage, e->stage_n[stage] - 1, 1)));
    *start_ms = a;
    *stop_ms = b;
    return CHD_OK;
}

chd_status chd_profile_get(chd_engine* e, int stage, double* total_ms, uint64_t* samples) {
    if (!e || stage < 0 || stage >= CHD_STAGE_COUNT || !total_ms || !samples) return CHD_ERR_INVALID;
    CHD_ENTER(e, ENTRY_COPY_WAIT);
    CU(e, cudaStreamSynchronize(e->stream));
    const uint64_t n = e->stage_n[stage];
    const uint64_t m = n < (uint64_t)chd_engine::EV_RING ? n : (uint64_t)chd_engine::EV_RING;
    double tot = 0;
    for (uint64_t i = n - m; i < n; i++) {
        float ms = 0;
        CU(e, cudaEventElapsedTime(&ms, e->evt(stage, i, 0), e->evt(stage, i, 1)));
        tot += ms;
    }
    *total_ms = tot;
    *samples = m;
    return CHD_OK;
}
}  // extern "C"
