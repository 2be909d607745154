// chd_engine.h — internal: the engine object behind include/chd_gpu.h and the helpers its translation units share.
// Layout of the host code (all device buffers are allocated once in chd_create; the tick path allocates nothing and —
// apart from chd_summary / the chd_get_* copies — never synchronises with the host):
//   chd_engine.cu    create / destroy, streams, memory, the prefetch protocol, CUDA-graph stage cache, instrumentation
//   chd_entities.cu  positions, cell assignment, spatial-hash build, the cell sort (chd_cell_sort)
//   chd_interest.cu  subscribers (lifecycle), query batches, QueryChannelIds, interest update
//   chd_tick.cu      emit, fan-out, channel start times, prefetch adoption, the batched tick and its two-stream choreography, summary
//   chd_rings.cu     update rings: host-owned snapshots, prefetched sets, device-owned rings with or without bytes, read-back
//   chd_results.cu   getters, chd_fetch_results, device views
//   chd_shard.cu     multi-GPU X-slabs: border export, halo import, the NCCL exchange
//   chd_extras.cu    window classes, ADJACENT_CHANNELS broadcast sets, config-plane helpers
//   chd_table.cu     the mode and call-order rules; entity-table mode: spawn / move / despawn by id, the id-valued results
//   chd_follow.cu    followers: slot -> entity bindings and the query batch generated from them
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "chd_scan.cuh"
#include "chd_types.cuh"

using namespace chd;

// One kind of per-tick input (positions, queries, rings) that a pipelined host uploads on up_stream into one of two staging sets
// while a tick is in flight, and hands to the next tick with chd_adopt_prefetched.  The sets' buffers stay with their kind; this
// holds which set is free, which is staged and which is read, and the events that order the uploads against the reads.  A
// prefetch fills the set other than the one adopted last, after the last recorded read of it (chd_pf_*).
// A double-buffered kind's sets are reached only through its Prefetch: readers use set `cur`, the writer uses the set that
// chd_pf_begin returned.  No member of chd_engine points into a set.
struct Prefetch {
    int next = 0;      // the set the next prefetch fills
    int staged = -1;   // the set holding an upload not adopted yet (-1: none)
    int cur = -1;      // the set the engine reads now (-1: none; positions: the front pair, never none)
    bool wait = false;  // the reader of `cur` has not been ordered after its upload yet
    cudaEvent_t ev_upload = nullptr, ev_read[2] = {nullptr, nullptr};
    bool read_recorded[2] = {false, false};
};

// One stable LSD radix sort by cell (chd_cell_sort), allocated by chd_create: the [digit][block] histogram, one look-back scan
// site per pass, the grid and pass 0's output when the sort takes two passes.
struct CellSort {
    uint32_t* hist = nullptr;  // [BUILD_MAX_BINS * blocks + 2]
    ScanSite site[2] = {};
    uint32_t blocks = 0;
    // true: every launch runs all `blocks` blocks, idle ones included (the pair grouping); false: only the blocks whose slice
    // starts below the length (the entity build)
    bool whole_grid = false;
    uint32_t *tmp_key = nullptr, *tmp_val = nullptr;
};

// Everything the visible-list copy kernels read besides the pairs: the cell CSR of a build and the emit preparation's outputs.
// Two sets, so that the next tick's build and preparation write one while the copy kernel of this tick still reads the other.
struct CopySet {
    uint32_t *sorted_ent = nullptr, *sorted_id = nullptr;  // sorted_id: entity-table mode only (chd_entity_table_init)
    uint32_t* cell_start = nullptr;                        // [C+2]
    uint64_t* voff = nullptr;
    uint32_t* first_pair = nullptr;
    TileDesc* tile_desc = nullptr;  // per-tile copy descriptors (chd_emit.cuh)
    uint32_t *general_tiles = nullptr, *n_general = nullptr;  // tiles with more than two segments: list, {length, consumer ticket}
    unsigned long long* n_visible = nullptr;  // V of this set's preparation (the summary keeps its own copy in Counters)
};

// One pair of position buffers: chd_create allocates set 0, the first chd_prefetch_entities set 1.
struct PosSet {
    double *x = nullptr, *z = nullptr;
    uint32_t n = 0;  // entities a prefetch uploaded into it
};

// Positions as the kernels read them (chd_positions).
struct Positions { const double *x = nullptr, *z = nullptr; };

struct chd_engine {
    chd_grid_cfg cfg;
    chd_limits lim;
    GridDev g;
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    // Guards (a) the shared query scratch between the stateless query entry points and the interest update and (b) a CUDA
    // graph capture on `stream` against launches of the stateless entry points, which may run on other threads.
    std::recursive_mutex mu;
    mutable std::string err;
    // what chd_destroy releases: device memory (dalloc), every stream but `stream` (chd_make_stream), every event but the
    // profiling ring (chd_make_event); each GraphSlot releases its own executable
    std::vector<void*> allocs;
    std::vector<cudaStream_t> streams;
    std::vector<cudaEvent_t> events;
    int sm_count = 132;
    int l2_bytes = 50 << 20;  // both read from the device in chd_create
    uint64_t n_launch = 0;  // kernels launched by this engine (bench.py reports it as gpu_launches)
    // CUDA graphs: the launch-bound small-kernel stages are captured per key and replayed (run_stage).  A slot holds one key:
    // pending (exec == nullptr) or captured; key 0 marks a free slot.
    struct GraphSlot {
        cudaGraphExec_t exec = nullptr;
        uint64_t key = 0;
        uint64_t nodes = 0;
        uint64_t used = 0;  // GraphSet::clock at this slot's last lookup
        GraphSlot() = default;
        GraphSlot(const GraphSlot&) = delete;
        GraphSlot& operator=(const GraphSlot&) = delete;
        ~GraphSlot() { release(); }
        void release() {
            if (exec) cudaGraphExecDestroy(exec);
            exec = nullptr;
        }
    };
    struct GraphSet {  // the graphs of one run_stage call site
        GraphSlot slot[8];
        uint64_t clock = 0;
    };
    bool use_graphs = true;
    cudaStream_t aux_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_interest = nullptr, ev_pairs = nullptr;
    bool interest_pending = false, pending_fanout = false;  // chd_begin_interest issued, not yet joined by chd_tick
    GraphSet g_build, g_build_b, g_interest, g_interest_b, g_emit_prep, g_fanout, g_export, g_import;
    uint64_t graph_launches = 0, graph_captures = 0;
    int64_t* d_time = nullptr;      // [0] = now_ns of the last update_interest, [1] = t_ns of the last fanout_tick
    // optional per-stage CUDA-event timing (chd_profile_*): [stage][0=start,1=stop]
    int profiling = 0;  // 0 off, 1 every stage, 2 the emit kernel only
    static constexpr int EV_RING = 1024;
    cudaEvent_t* ev = nullptr;  // [CHD_STAGE_COUNT][EV_RING][2]
    uint64_t stage_n[CHD_STAGE_COUNT] = {};
    cudaEvent_t& evt(int stage, uint64_t i, int which) { return ev[((size_t)stage * EV_RING + (size_t)(i % EV_RING)) * 2 + which]; }

    // ---- entities
    uint32_t n_own = 0, n_halo = 0;  // entities with positions / appended halo records
    bool halo_on_device = false;     // multi-GPU: the build length (own + halo) lives in d_n_build
    uint32_t* d_n_build = nullptr;
    bool have_gid = false;
    // position pairs: the set calls, chd_entity_buffers and the table-mode kernels use the front pair pos[pf_pos.cur] (chd_pos_front;
    // chd_create makes it 0), a prefetch fills the back one and chd_adopt_prefetched makes it the front one
    PosSet pos[2];
    Prefetch pf_pos;
    Positions in_place;  // the caller's device arrays the last set call reads in place (x == nullptr: the front pair)
    float* d_pos_f32[2] = {nullptr, nullptr};  // float staging of chd_set_entities_f32 [0] / chd_prefetch_entities_f32 [1]: x then z
    cudaStream_t up_stream = nullptr;  // every prefetch upload
    uint32_t *d_gid = nullptr;            // [max_entities] global ids (multi-GPU) of own + halo
    uint32_t *d_key = nullptr, *d_prev_key = nullptr;  // [max_entities] cell key per entity
    // the build's sort by cell: 4 blocks per SM, N-sized temporaries, which chd_get_rehome and chd_handoff_entities borrow as
    // scratch between builds
    CellSort ent_sort;
    uint32_t* d_sorted_key = nullptr;
    // Readers use copy_set[pf_copy.cur] (chd_copy_in).  Each build writes the set the last copy kernel did not read (chd_pf_begin
    // orders the build after the last copy that read it) and adopts it when it ends; chd_pf_note_read records each copy kernel's read.
    CopySet copy_set[2];
    Prefetch pf_copy;
    // Two-stream ticks: the build runs on build_stream (highest priority), the copy kernel on copy_stream (lowest priority), so
    // that the next tick's head runs beside it.  copy_pending: the set read by a copy kernel on copy_stream that the engine stream
    // is not ordered after yet (-1: none; chd_copy_wait).
    cudaStream_t build_stream = nullptr, copy_stream = nullptr;
    int copy_pending = -1;
    // one look-back scan site per call site: stages run concurrently on two streams and must not share scan state
    unsigned long long* d_epoch = nullptr;  // [EP_COUNT] stage epochs for the look-back scans
    ScanSite site_qoff{}, site_slot{}, site_voff{}, site_border{};
    uint64_t stage_execs[10] = {};  // [EP_COUNT]
    std::vector<ScanSite*> sites;  // every scan site (chd_make_site registers them)
    bool assigned = false, built = false, have_prev_key = false, entities_dirty = false;
    uint32_t n_sorted = 0;
    bool sorted_dev_n = false;  // the last build's length was d_n_build (own + halo on the device), not n_sorted
    // handover
    uint32_t *d_ho_entity = nullptr, *d_ho_src = nullptr, *d_ho_dst = nullptr;
    uint32_t ho_cap = 0;

    // ---- subscribers / pairs
    uint32_t n_slots = 0;
    uint32_t* d_conn = nullptr;
    // lifecycle: pending per-slot changes (SLOT_*), applied by the next interest update; source record of an immigrant;
    // staging for the slot / connection-id lists of chd_add_subscribers / chd_remove_subscribers / chd_migrate_*
    uint8_t* d_slot_ctl = nullptr;
    uint32_t *d_slot_src = nullptr, *d_lc_slot = nullptr, *d_lc_aux = nullptr;
    bool lifecycle_used = false;  // the interest kernels look at d_slot_ctl only once a lifecycle call has been made
    MigView mig{nullptr, 0, 0, 0};  // gathered migration blobs of this tick (chd_shard.cu)
    PairBuf pairs[2];
    int cur = 0;
    // ---- query scratch
    struct QStage {
        uint32_t *sub; uint8_t* kind;
        double *sph_cx, *sph_cz, *sph_r, *box_cx, *box_cz, *box_ex, *box_ez, *cone_cx, *cone_cz, *cone_dx, *cone_dz, *cone_angle, *cone_r;
        uint32_t *spot_off, *spot_ndist; double *spot_x, *spot_z; uint32_t* spot_dist;
        QueryDev view;   // a prefetch set: the batch it holds
        uint32_t spots;  // and its spot total
    } dq{};
    // chd_prefetch_queries: two staging sets, allocated by the first prefetch that fills them.
    // pf_q.cur: the adopted batch the next interest update with q == NULL consumes (-1 once consumed).
    QStage dq_pf[2] = {};
    Prefetch pf_q;
    Bbox* d_bbox = nullptr;
    uint32_t *d_window = nullptr, *d_side_cell = nullptr, *d_side_dist = nullptr, *d_side_cnt = nullptr;
    uint64_t* d_win_off = nullptr;
    uint32_t *d_status = nullptr, *d_qcount = nullptr;
    uint32_t* d_qstatus = nullptr;              // statuses of the stateless query path (chd_query_channel_ids)
    unsigned long long* d_win_cursor = nullptr;  // bump cursor of the window scratch (zeroed by the stage's first kernel)
    uint32_t* d_noff = nullptr;                 // [S+1] new pair offsets, scanned into scratch: the interest update is transactional
    uint64_t* d_qoff = nullptr;  // stateless query CSR offsets
    uint32_t *d_qout_id = nullptr, *d_qout_dist = nullptr;
    int32_t* d_slot_query = nullptr;
    uint32_t last_nq = 0;
    // diff
    uint32_t *d_new_off = nullptr;  // scratch for u64 -> u32 offset narrowing (stateless query path)
    uint32_t *d_new_sub = nullptr, *d_new_ch = nullptr, *d_gone_sub = nullptr, *d_gone_ch = nullptr;
    // emit
    uint32_t *d_vcnt = nullptr, *d_vis = nullptr;
    uint32_t* d_pair_ch = nullptr;  // channel id of every current pair (written by interest_fill_kernel)
    // ---- window classes of the due list (chd_due_classes): keys written by the fan-out kernel, scratch allocated on first use
    DueKey* d_due_key = nullptr;
    uint32_t *d_cls_table = nullptr, *d_cls_slot = nullptr, *d_cls_rep = nullptr, *d_cls_cnt = nullptr, *d_cls_flag = nullptr, *d_cls_rank = nullptr,
             *d_cls_of = nullptr, *d_cls_out_rep = nullptr, *d_cls_out_cnt = nullptr;
    uint32_t cls_table_size = 0;
    ScanSite site_class{};
    // ---- ADJACENT_CHANNELS broadcast sets (chd_adjacent_broadcast): scratch allocated on first use, grown on demand
    uint8_t* d_conn_type = nullptr;
    bool have_conn_type = false, by_cell_valid = false;
    uint32_t *d_bc_in = nullptr, *d_bc_cnt = nullptr, *d_bc_off = nullptr, *d_bc_msgoff = nullptr, *d_bc_out = nullptr;
    uint64_t bc_msg_cap = 0, bc_out_cap = 0;
    ScanSite site_bcast{};
    bool pair_ch_valid = false;
    // ---- payload assembly + framing (chd_payload.cu): optional stage, buffers grown on demand
    struct Payload {
        uint64_t *d_entry_off = nullptr, *d_full_off = nullptr, *d_cls_off = nullptr, *d_conn_off = nullptr;
        uint8_t *d_entry_bytes = nullptr, *d_full_bytes = nullptr, *d_url = nullptr, *d_blob = nullptr, *d_out = nullptr, *d_stage = nullptr, *d_comp = nullptr;
        uint32_t *d_cls_len = nullptr, *d_fc_cnt = nullptr, *d_fc_off = nullptr, *d_fc_cursor = nullptr, *d_fc_idx = nullptr, *d_conn_cap = nullptr,
                 *d_conn_len = nullptr, *d_conn_frames = nullptr, *d_ndrop = nullptr;
        uint64_t cap_entry_off = 0, cap_entry_bytes = 0, cap_full_off = 0, cap_full_bytes = 0, cap_url = 0, cap_cls = 0, cap_cls_off = 0, cap_blob = 0,
                 cap_fc = 0, cap_fc_off = 0, cap_fc_cur = 0, cap_fc_idx = 0, cap_conn_cap = 0, cap_conn_off = 0, cap_conn_len = 0, cap_conn_frames = 0,
                 cap_comp = 0, cap_ndrop = 0, cap_out = 0, cap_stage = 0, cap_site_cls = 0, cap_site_fc = 0, cap_site_conn = 0;
        ScanSite site_cls{}, site_fc{}, site_conn{};
        uint32_t url_len = 0, msg_type = 8, n_entries = 0, n_classes = 0;
        uint64_t blob_len = 0;
        bool have_input = false, assembled = false;
    } pl;
    // chd_fetch_results reads back on its own stream as soon as the aux chain (pairs, diff, due list) and the emit
    // preparation (visible offsets) are done, i.e. while the emit kernel is still streaming
    cudaStream_t dl_stream = nullptr, dl_stream_b = nullptr;  // phase A / phase B of the early read-back
    cudaEvent_t ev_prep_done = nullptr, ev_build_done = nullptr;
    // ev_counts: the cell CSR offsets of the build in flight are final (recorded between the two halves of a single-pass build);
    // prep_stream: where the emit preparation runs when it overlaps the build's scatter
    cudaEvent_t ev_counts = nullptr;
    cudaStream_t prep_stream = nullptr;
    bool build_done_recorded = false;  // this tick ran a build (its end is ev_build_done)
    // chd_fetch_results_async: completion events of the two copy phases; the next tick is ordered after them on the device
    // (two fetches may be outstanding: the host waits for tick k-1 after it has enqueued tick k and its fetch)
    cudaEvent_t ev_fetch_a[2] = {nullptr, nullptr}, ev_fetch_b[2] = {nullptr, nullptr};
    // chd_fetch_results_async is two hops: result arrays -> a device-side snapshot (ev_fetch_a/b: the next tick may overwrite the
    // arrays) -> pinned host memory at PCIe speed on its own stream (ev_fetch_done: chd_fetch_wait)
    cudaEvent_t ev_fetch_done[2] = {nullptr, nullptr};
    cudaStream_t dl_stream_c = nullptr;
    uint8_t* d_fetch_stage[2] = {nullptr, nullptr};
    uint64_t fetch_stage_bytes[2] = {0, 0};
    void* fetch_header[2] = {nullptr, nullptr};
    // the visible delta of fetch set fi: deltas it carries (0: none or no delta buffers) and n_slots; dl_stream_d: its snapshot hop
    uint32_t fetch_deltas[2] = {0, 0}, fetch_delta_slots[2] = {0, 0};
    cudaStream_t dl_stream_d = nullptr;
    uint64_t fetch_issued = 0, fetch_waited = 0;
    bool fetch_guard = false;
    bool early_ready = false;  // ev_join + ev_prep_done of the last tick are recorded
    uint64_t* d_vis_off = nullptr;
    uint64_t max_tiles = 0;
    uint64_t vis_estimate = 0;  // n_visible of the last summary the host decoded (0 = none yet): sizes the emit grid
    // ---- update rings (chd_rings.cu): host-owned (one tick's CSR by cell: chd_set_rings, chd_prefetch_rings) or device-owned
    // (chd_rings_init: ChannelData.OnUpdate on the GPU, data.go:149-173)
    struct Rings {
        struct RStage {
            uint32_t *off = nullptr, *sender = nullptr; int64_t* arrival = nullptr; uint64_t *index = nullptr, *cmi = nullptr;
            uint32_t total = 0;    // entries uploaded
            bool has_cmi = false;  // cmi holds a channel_msg_index
        };
        // set: chd_set_rings' staging (chd_create); on device-owned rings arrival / sender / index are the entry slabs and cmi is
        // ChannelData.msgIndex.  pf_set: chd_prefetch_rings' two sets, allocated by the first prefetch that fills them; pf.cur is
        // the set `view` reads (-1: the rings came from chd_set_rings / chd_rings_init).
        RStage set, pf_set[2];
        Prefetch pf;
        // device-owned rings: per-cell begin / end cursors into slabs of `cap` entries inside set.arrival / set.sender / set.index;
        // the updates of one append (upd_off: CSR by cell), grown on demand; the read-back's live-entry CSR and its scan scratch
        bool owned = false;
        uint32_t cap = 0;
        uint32_t *begin = nullptr, *end = nullptr, *upd_off = nullptr, *upd_sender = nullptr, *flat_off = nullptr, *scan_scratch = nullptr;
        int64_t* upd_arrival = nullptr;
        uint64_t upd_arrival_cap = 0, upd_sender_cap = 0;
        // a communicator engine's chd_rings_append only uploads its updates into upd_*: chd_tick_sharded appends them after the
        // ring-limit import (rule 12)
        bool staged = false;
        uint32_t staged_updates = 0;
        // rule 14: an append was made since chd_rings_init (the byte reservation comes before it); an append was applied, or the
        // rings were emptied, after the last fan-out pass (chd_assemble_payloads replays that pass's windows over the rings it read)
        bool appended = false, after_fanout = false;
        // byte-carrying device rings (include/chd_gpu_ring_bytes.h, allocated by chd_rings_reserve_bytes): each cell's slab of
        // per_cell bytes in `slab`, every entry slot's byte position (relative to its cell's slab) and length beside set.arrival, each
        // cell's live byte range (bb, be) in `cur`; the staged bytes of an append (upd_boff: [n_updates + 1] offsets into upd_bytes)
        struct RingBytes {
            bool on = false;
            uint32_t per_cell = 0;
            uint8_t *slab = nullptr, *upd_bytes = nullptr;
            uint32_t *pos = nullptr, *len = nullptr, *cur = nullptr;
            unsigned long long* upd_boff = nullptr;
            uint64_t upd_boff_cap = 0, upd_bytes_cap = 0;
        } bytes;
        // the rings the kernels read (chd_ring_view adds `start`): `set`, the caller's device arrays (zero-copy), an adopted prefetch set
        // or the device-owned rings; d_total their entry count, written for host-owned rings by the next pass that reads them, on its
        // stream (chd_ring_total_flush): a kernel on the engine stream between ticks would queue behind the copy kernel's grid
        RingDev view{};
        uint32_t* d_total = nullptr;
        uint32_t total = 0;
        bool total_pending = false;
    } rings;
    uint32_t* d_cell_max_interval = nullptr;  // [C] ChannelData.maxFanOutIntervalMs (subscription.go:84-86)
    // ring limits on slabs (include/chd_gpu_rings.h), allocated by their first use: the exported shadow of d_cell_max_interval [C],
    // the record count of an export through chd_export_ring_limits, the export compaction's scan site
    uint32_t *d_ring_lim_x = nullptr, *d_ring_lim_n = nullptr;
    ScanSite site_ring_lim{};
    int64_t* d_cell_start_ns = nullptr;       // [C] per-channel ChannelTime origin (chd_set_channel_start_times) or nullptr
    bool have_cell_start = false;

    uint32_t* d_by_cell = nullptr;  // pairs grouped by cell
    CellSort pair_sort;             // its sort: one block per tile of max_pairs, at most 4096; P-sized temporaries
    chd_due* d_due = nullptr;
    // counters
    Counters* d_ctr = nullptr;
    Counters* h_ctr = nullptr;  // pinned
    // multi-GPU exchange (chd_comm_init): NCCL communicator (opaque here), engine-owned record buffers
    void* comm = nullptr;
    int comm_rank = 0, comm_world = 1;
    uint32_t border_cap = 0;
    uint32_t rec_per_rank = 0;        // border records per rank in the gathered buffer (0: plain contiguous records)
    uint64_t rec_stride_words = 0;    // words one rank contributes to the all-gather (border records + migration blob)
    uint32_t mig_subs = 0, mig_pairs = 0;  // migration blob capacities (0: no subscriber migration)
    bool mig_packed = false;          // chd_migrate_out was called for the coming tick
    // the ring-limit section of a contribution (after the migration blob): its word offset and its record capacity, the largest
    // served-cell count of any rank.  Layout: [count, 3 words of padding, 2 x u32 per record]
    uint64_t ring_sec_off = 0;
    uint32_t ring_sec_cap = 0;
    uint32_t *d_rec_local = nullptr, *d_rec_all = nullptr;
    unsigned long long* assign_bump = nullptr;  // epoch the next assign_cells_kernel launch bumps for its caller (border export)
    // peer exchange (chd_shard.cuh): this rank's window, the peers' windows mapped with CUDA IPC, device-side sequence / counts
    bool peer_push = false, peer_mapped = false;
    uint32_t* d_peer_win = nullptr;
    void* peer_base[16] = {};
    unsigned long long* d_xchg_seq = nullptr;
    uint32_t *d_push_done = nullptr, *d_peer_count = nullptr;
    uint64_t xchg_seq = 0;  // host mirror of the device sequence (selects the window buffer a graph variant is captured for)
    uint64_t n_collectives = 0;
    // border export scratch
    uint32_t *d_bflag = nullptr, *d_boff = nullptr;
    uint32_t* h_u32 = nullptr;  // pinned scalar
    // scratch of the tick driver's getters (chd_get_visible*, export counts): separate from h_u32, which the stateless entry
    // points use under the engine mutex from other threads
    uint32_t* h_get = nullptr;
    // ---- visible-set deltas (chd_delta.cu): everything is allocated by the first chd_reserve_visible_delta(_ids)
    struct Delta {
        bool on = false;
        // id mode (chd_reserve_visible_delta_ids): entities are named by global id; snap_key and now_gkey are indexed by it
        bool ids = false;
        uint32_t id_space = 0;
        uint32_t* now_gkey = nullptr;  // [id_space] cell of each id in the last build, 0xFFFFFFFF = absent
        uint32_t* bad_ids = nullptr;   // [1] the last id-mode delta met an id >= id_space or a duplicate (CHD_OVF_DELTA_IDS)
        uint32_t *snap_key = nullptr, *snap_cell_start = nullptr, *snap_sorted = nullptr, *snap_pair_off = nullptr, *snap_pair_cell = nullptr;
        uint32_t* snap_hdr = nullptr;  // [0] entity count, [1] slot count of the snapshot
        uint32_t *arr_rank = nullptr, *dep_rank = nullptr, *arr = nullptr, *dep = nullptr, *arr_start = nullptr, *dep_start = nullptr;
        uint32_t *cnt_enter = nullptr, *cnt_leave = nullptr;
        uint64_t *enter_off = nullptr, *leave_off = nullptr;
        uint32_t *enter = nullptr, *leave = nullptr;
        uint64_t enter_cap = 0, leave_cap = 0;
        uint32_t n_out = 0;  // slots the output CSRs cover: max(slots now, slots at any earlier delta) (never shrinks)
        ScanSite site_arr{}, site_dep{}, site_enter{}, site_leave{};
        GraphSet g;
        cudaEvent_t ev_in = nullptr, ev_done = nullptr;  // two-stream tick: the build is done / the delta is done
        bool done_recorded = false;  // the last tick ran the delta off the engine stream: its end (and CHD_OVF_DELTA) is ev_done
        // read-back (chd_fetch_results*_delta): deltas enqueued (seq) and seq at the last fetch; ev_end: recorded after every delta on
        // its stream.  ev_read[fi]: fetch set fi's snapshot of the lists is done; the next delta waits for the latest (read_guard).
        uint64_t seq = 0, fetched = 0;
        cudaEvent_t ev_end = nullptr, ev_read[2] = {nullptr, nullptr};
        bool read_guard = false;
        int read_fi = 0;
    } dl;
    // chd_set_slab / chd_set_entity_ids / chd_comm_init were used: halo indices are not stable, no index-mode deltas (id mode is
    // not affected).  Sticky: chd_set_entity_ids(NULL) leaves no other trace, so this cannot be derived from have_gid / slab.
    bool delta_blocked = false;
    // chd_set_slab (directly or through chd_comm_init) made this engine an X-slab: the multi-GPU calls work in entity-table mode
    // only on such an engine, made a slab before chd_entity_table_init
    bool slab = false;
    // ---- entity-table mode (chd_table.cu): entities spawned / moved / despawned by id; everything is allocated by
    // chd_entity_table_init.  Slots are position indices; n_own is the high-water mark.
    struct Table {
        bool on = false;
        std::unordered_map<uint32_t, uint32_t> slot_of;  // live id -> slot
        std::deque<uint32_t> free_fifo;                  // released slots, reused first in, first out
        struct Held {
            uint32_t slot;
            uint64_t build;  // the first build that sees the slot empty: released by a successful delta of that build or a later one
        };
        std::deque<Held> quarantine;
        uint32_t hw = 0;       // slots [0, hw) have been used
        uint32_t bits = 0;     // the device table has 2^bits words
        uint64_t used = 0;     // live entries + tombstones in the device table
        uint64_t rebuilds = 0, builds = 0;  // builds: table-mode builds so far (the device counts them too: d_build_seq)
        bool ho_raw = false;   // the handover list holds slots of a fresh cell assignment (chd_assign_host)
        uint64_t* d_table = nullptr;
        uint32_t *d_id_of_slot = nullptr, *d_snap_id = nullptr, *d_winner = nullptr, *d_mslot = nullptr;
        uint32_t *d_ho_tmp = nullptr, *d_build_seq = nullptr;  // d_build_seq[0] = builds, [1] = stashed handover count
        uint8_t* d_flag = nullptr;                             // slot spawned / despawned since the last cell assignment
        unsigned long long* d_stats = nullptr;                 // moves applied, to unknown ids, superseded within a call
        uint32_t* d_ev = nullptr;   // event staging: [N] ids, [N] slots
        double* d_ev_pos = nullptr;  // [2N] x, z (moves: f64, or f32 in the first half)
        // spawn / despawn uploads go through two pinned buffers, each reused once the copy made from it two calls ago is done
        uint8_t* h_stage[2] = {nullptr, nullptr};
        uint64_t h_stage_cap[2] = {0, 0};
        cudaEvent_t ev_stage[2] = {nullptr, nullptr};
        int next_stage = 0;
        GraphSet g_post;
        // facings (include/chd_gpu_facing.h), allocated by the first facing call: d_fx / d_fz [N] per slot (0, 0: none), written by
        // the event kernels and read by the follow stage, both on the engine stream; d_ev_face: [2N] staging of the events' facings
        double *d_fx = nullptr, *d_fz = nullptr, *d_ev_face = nullptr;
    } tbl;
    // ---- followers (chd_follow.cu): everything is allocated by the first chd_follow_bind
    struct Follow {
        bool on = false;
        std::vector<uint8_t> h_kind;  // host mirror of st.kind (0: the slot follows nothing): argument checks, counts
        uint32_t n_bound = 0;
        FollowDev st{};     // per-slot bindings, [max_subscribers]
        FollowBatch q{};    // the generated batch, [max_queries]; q.n_selected: queries in it
        uint8_t* spot_buf = nullptr;  // merged batches: q.spot_x | q.spot_z | q.spot_dist, spot_cap spots each, grown on demand
        uint64_t spot_bytes = 0, spot_cap = 0;
        uint32_t* hdr = nullptr;  // [1] the host part's length, written before the merged generation's graph
        QueryDev view{};    // the generated batch as the interest stage reads it
        bool ready = false;     // a generated batch waits for the interest update that consumes it
        uint8_t* d_stage = nullptr;  // chd_follow_bind / chd_follow_unbind: staged arguments
        uint64_t stage_cap = 0;
        uint32_t *g_slot = nullptr, *g_entity = nullptr, *g_status = nullptr, *g_count = nullptr;  // chd_get_follow's lists, [max_queries]
        double *g_cx = nullptr, *g_cz = nullptr;
        ScanSite site{};
        GraphSet g;
        // frames (chd_follow_set_frame): device state allocated by the first frame; h_frame mirrors fr.on; n_framed counts the bound
        // followers with a frame, and the generation runs the Frame instantiations only while it is not zero
        FollowFrame fr{};
        std::vector<uint8_t> h_frame;
        uint32_t n_framed = 0;
        uint32_t* g_fslot = nullptr;  // chd_get_follow_frame's lists: [max_queries] slots, [6][max_queries] doubles
        double* g_fval = nullptr;
    } fw;
    // ---- explicit subscriptions (chd_subs.cu): scratch allocated on first use, op arrays grown on demand
    struct Subs {
        uint64_t op_cap = 0;  // ops every op array below holds
        uint32_t *slot = nullptr, *channel = nullptr, *interval = nullptr;
        int32_t* delay = nullptr;
        uint8_t *op = nullptr, *present = nullptr, *skip_self = nullptr, *skip_first = nullptr, *status = nullptr;
        // sort keys and values (first pass by cell, second by slot), each op's slot (S if rejected) and cell index
        uint32_t *key = nullptr, *key_out = nullptr, *idx1 = nullptr, *idx2 = nullptr, *eff_slot = nullptr, *cell = nullptr;
        uint32_t *beg = nullptr, *cnt = nullptr, *noff = nullptr;  // [max_subscribers (+2)]: per touched slot its first op / new run length
    } subs;

    bool fail(const char* fmt, ...) const {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof buf, fmt, ap);
        va_end(ap);
        err = buf;
        return false;
    }
};

#define CU(e, call)                                                                                  \
    do {                                                                                             \
        cudaError_t _r = (call);                                                                     \
        if (_r != cudaSuccess) {                                                                     \
            (e)->fail("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_r), __FILE__, __LINE__);   \
            return CHD_ERR_CUDA;                                                                     \
        }                                                                                            \
    } while (0)

// one kernel launch precedes every KCHECK; scans report their own launch count through SCAN()
#define KCHECK(e)                    \
    do {                             \
        (e)->n_launch++;             \
        CU(e, cudaGetLastError());   \
    } while (0)
#define SCAN(e, ...)                                  \
    do {                                              \
        (e)->n_launch += (uint64_t)(__VA_ARGS__);     \
        CU(e, cudaGetLastError());                    \
    } while (0)

// What an entry point of include/chd_gpu.h needs before it touches the engine.  Each one declares it once, with CHD_ENTER after
// its argument and mode-rule checks, and the steps always run in the order of the list:
//   ENTRY_LOCK         holds e->mu until the entry point returns: the entry points that may run on any thread (chd_cell_of*,
//                      chd_query_channel_ids, chd_adjacent_broadcast) and those that share state with them: h_u32, the query
//                      scratch, the engine stream while a graph is being captured (run_stage).
//   ENTRY_DEVICE       makes e->device the calling thread's current device: every entry point that makes a CUDA call.
//   ENTRY_COPY_WAIT    chd_copy_wait: every entry point that reads the expanded list, hands out device memory, rewrites something
//                      the pending copy kernel reads or is a documented completion point (chd_sync, chd_summary, the getters).
//   ENTRY_FETCH_GUARD  chd_fetch_guard on the engine stream: every entry point that rewrites arrays an outstanding asynchronous
//                      read-back may still be copying.
// COPY_WAIT and FETCH_GUARD imply DEVICE, and CHD_ENTER(e, 0) marks an entry point that needs none.  A failed step returns CHD_ERR_CUDA.
enum : unsigned { ENTRY_DEVICE = 1, ENTRY_LOCK = 2, ENTRY_COPY_WAIT = 4, ENTRY_FETCH_GUARD = 8 };
chd_status chd_enter(chd_engine* e, unsigned needs, std::unique_lock<std::recursive_mutex>& lock);  // CHD_ENTER's steps
#define CHD_ENTER(e, needs)                                   \
    std::unique_lock<std::recursive_mutex> chd_entry_lock_;   \
    if (const chd_status chd_entry_st_ = chd_enter((e), (needs), chd_entry_lock_); chd_entry_st_ != CHD_OK) return chd_entry_st_

struct StageTimer {  // records a CUDA-event pair around a stage on stream `s` when profiling is on
    chd_engine* e;
    cudaStream_t s;
    int stage;
    bool on;
    StageTimer(chd_engine* e_, cudaStream_t s_, int stage_)
        : e(e_), s(s_), stage(stage_), on(e_->profiling == 1 || (e_->profiling == 2 && stage_ == CHD_STAGE_EMIT_KERNEL)) {
        if (on) cudaEventRecord(e->evt(stage, e->stage_n[stage], 0), s);
    }
    ~StageTimer() {
        if (on) {
            cudaEventRecord(e->evt(stage, e->stage_n[stage], 1), s);
            e->stage_n[stage]++;
        }
    }
};

template <typename T>
static bool dalloc(chd_engine* e, T** p, uint64_t count) {
    void* q = nullptr;
    const uint64_t bytes = (count ? count : 1) * sizeof(T);
    cudaError_t r = cudaMalloc(&q, bytes);
    if (r != cudaSuccess) {
        e->fail("cudaMalloc(%llu bytes) failed: %s", (unsigned long long)bytes, cudaGetErrorString(r));
        return false;
    }
    e->allocs.push_back(q);
    *p = (T*)q;
    return true;
}

// Every secondary stream: non-blocking, at the device's highest priority so that its short kernels and copies do not queue
// behind the emit kernel's grid, or at the lowest (`lowest`: the copy stream, whose grid yields to the next tick's head).
// chd_destroy releases it.
static inline bool chd_make_stream(chd_engine* e, cudaStream_t* s, bool lowest = false) {
    int lo = 0, hi = 0;
    cudaError_t r = cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (r == cudaSuccess) r = cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, lowest ? lo : hi);
    if (r != cudaSuccess) return e->fail("cudaStreamCreateWithPriority failed: %s", cudaGetErrorString(r));
    e->streams.push_back(*s);
    return true;
}

// An ordering-only event (no timing); chd_destroy releases it.
static inline bool chd_make_event(chd_engine* e, cudaEvent_t* ev) {
    cudaError_t r = cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
    if (r != cudaSuccess) return e->fail("cudaEventCreateWithFlags failed: %s", cudaGetErrorString(r));
    e->events.push_back(*ev);
    return true;
}

// one query staging set: chd_create's dq, chd_prefetch_queries' dq_pf[]
static inline bool alloc_qstage(chd_engine* e, chd_engine::QStage& qs) {
    const uint64_t Q = e->lim.max_queries, SP = e->lim.max_spots;
    return dalloc(e, &qs.sub, Q) && dalloc(e, &qs.kind, Q) && dalloc(e, &qs.sph_cx, Q) && dalloc(e, &qs.sph_cz, Q) && dalloc(e, &qs.sph_r, Q) &&
           dalloc(e, &qs.box_cx, Q) && dalloc(e, &qs.box_cz, Q) && dalloc(e, &qs.box_ex, Q) && dalloc(e, &qs.box_ez, Q) &&
           dalloc(e, &qs.cone_cx, Q) && dalloc(e, &qs.cone_cz, Q) && dalloc(e, &qs.cone_dx, Q) && dalloc(e, &qs.cone_dz, Q) &&
           dalloc(e, &qs.cone_angle, Q) && dalloc(e, &qs.cone_r, Q) && dalloc(e, &qs.spot_off, Q + 1) && dalloc(e, &qs.spot_ndist, Q) &&
           dalloc(e, &qs.spot_x, SP) && dalloc(e, &qs.spot_z, SP) && dalloc(e, &qs.spot_dist, SP);
}

enum { EP_BUILD = 0, EP_QUERY, EP_EMIT, EP_FANOUT, EP_BORDER, EP_BCAST, EP_CLASS, EP_PAYLOAD, EP_DELTA, EP_FOLLOW, EP_COUNT };  // d_epoch has EP_COUNT slots
static_assert(EP_COUNT == sizeof(chd_engine::stage_execs) / sizeof(uint64_t), "one execution counter per stage epoch");

// ---- helpers shared by the translation units (C linkage only so that definitions may sit inside their extern "C" blocks)
extern "C" {
// epochs start at 1 so that the zero-initialised descriptors (epoch 0) read as stale on first use
bool chd_init_epochs(chd_engine* e);
bool chd_make_site(chd_engine* e, ScanSite& site, uint64_t n_max, int stage);
// Zero-copy inputs: a pointer into this device's memory is consumed in place (no staging copy); the caller keeps it valid
// and unmodified until the work that reads it has finished (chd_summary / chd_sync / any chd_get_*).
bool chd_is_device_ptr(const chd_engine* e, const void* p);
void chd_dfree(chd_engine* e, void* p);
// The prefetch protocol (struct Prefetch).  begin: creates up_stream and the events on first use, orders up_stream after the
// last recorded read of the set the prefetch fills and returns that set; the caller then enqueues the upload on up_stream.
// end: records the upload and stages the set (a second prefetch before an adoption refills it).  Both take the writer's stream
// instead of up_stream when one is given (the copy-input sets: the build writes them).  adopt: makes the staged set
// the one read (false: nothing staged).  wait: orders reader stream `s` after the upload, once per adoption.  note_read:
// records a read of `set` (-1: none) on `s`, outside any graph capture, so that no prefetch overwrites it before that read.
// after_read: orders `s` after the last recorded read of `set` (a writer of that set).
chd_status chd_pf_begin(chd_engine* e, Prefetch& p, int* set, cudaStream_t s = nullptr);
chd_status chd_pf_end(chd_engine* e, Prefetch& p, cudaStream_t s = nullptr);
bool chd_pf_adopt(Prefetch& p);
chd_status chd_pf_wait(chd_engine* e, Prefetch& p, cudaStream_t s);
chd_status chd_pf_note_read(chd_engine* e, Prefetch& p, int set, cudaStream_t s);
chd_status chd_pf_after_read(chd_engine* e, const Prefetch& p, int set, cudaStream_t s);
chd_status chd_read_u32(chd_engine* e, const uint32_t* d, uint32_t* v);
// Orders the engine stream after the copy kernel a two-stream chd_tick left running on copy_stream (device-side, no host sync).
// Which entry points call it: ENTRY_COPY_WAIT.
cudaError_t chd_copy_wait(chd_engine* e);
chd_status chd_decode_summary(chd_engine* e, chd_tick_summary* out);
chd_status chd_assign_cells_impl(chd_engine* e, cudaStream_t s);
// Host half of a cell assignment: the key buffers swap (handover detection compares against the keys of the previous
// assignment, same entity count; swapped, never copied) and the own entities count as assigned.  Returns the previous keys or
// nullptr.  A replayed assignment graph runs only the device half, so its caller runs this.
uint32_t* chd_assign_host(chd_engine* e);
// the current positions were replaced by n others (a set call, chd_set_entity_count, an adopted prefetch): nothing is assigned
// or built for them yet
void chd_entities_replaced(chd_engine* e, uint32_t n);
// Called on the host wherever a stage's epoch is about to be bumped on the device: every 2^20 executions of a stage the
// descriptors of its scan sites are cleared, so no descriptor can survive until the 22-bit epoch repeats.  `s` is the
// stream the stage runs on, so the clear is ordered before the stage's scans.
chd_status chd_epoch_tick(chd_engine* e, cudaStream_t s, int stage);
// lifecycle / migration calls may name slots beyond the current count: extends the slot table (new slots hold no pairs)
chd_status chd_grow_slots(chd_engine* e, uint32_t new_n);
chd_status chd_fetch_guard(chd_engine* e, cudaStream_t s);
// chd_build / chd_update_interest without the fetch guard, enqueued on `s` (chd_tick runs the interest update on aux_stream)
chd_status chd_build_on(chd_engine* e, cudaStream_t s);
chd_status chd_update_interest_on(chd_engine* e, cudaStream_t s, const chd_query_batch* q, int64_t now_ns);
// Copies a query batch into the engine's device SoA (or a prefetch staging set) on `s`, device arrays in place, and returns the
// device view; *spots (if given): the batch's spot total
chd_status chd_upload_queries(chd_engine* e, cudaStream_t s, const chd_query_batch* q, QueryDev* out, bool need_sub,
                              chd_engine::QStage* stage = nullptr, uint32_t* spots = nullptr);
// update rings (chd_rings.cu): what the kernels read; chd_create's and chd_adopt_prefetched's parts; the append kernel on `s` over
// n_updates updates already in rings.upd_* (and, on a byte-carrying engine, their bytes in rings.bytes.upd_*)
RingDev chd_ring_view(const chd_engine* e);
chd_status chd_ring_total_flush(chd_engine* e, cudaStream_t s);
chd_status chd_rings_create(chd_engine* e);
void chd_rings_adopt(chd_engine* e);
chd_status chd_rings_apply(chd_engine* e, cudaStream_t s, uint32_t n_updates);
// The stable sort by cell on `s` (chd_entities.cu): values val (nullptr: the index) of keys key[0, n) in [0, keys) (n_ptr: the
// live length on the device) into val_out, in <= 2 passes of <= 10-bit digits.  key_out: where a two-pass sort writes the sorted
// keys.  csr: the cell CSR to publish (nullptr: none).  bump: the epoch the first kernel opens.  assign: pass 0's histogram also
// assigns the keys.  part: 0 = the whole sort; single-pass sorts only: 1 = histogram, scan and cell CSR, 2 = scatter.
struct FusedAssign;
chd_status chd_cell_sort(chd_engine* e, cudaStream_t s, const CellSort& cs, uint32_t keys, const uint32_t* key, const uint32_t* val, uint32_t n,
                         const uint32_t* n_ptr, uint32_t* key_out, uint32_t* val_out, const ScatterExtras* csr = nullptr,
                         unsigned long long* bump = nullptr, const FusedAssign* assign = nullptr, int part = 0);
// the visible-set delta stage on `s` (chd_delta.cu)
chd_status chd_delta_on(chd_engine* e, cudaStream_t s);
// The last visible delta's list lengths and its id-mode error flag (CHD_OVF_DELTA_IDS), read on `s` once the delta has finished
// there: one host round trip (chd_delta.cu)
struct DeltaLengths {
    uint64_t n_entered, n_left;
    bool bad_ids;
};
chd_status chd_read_delta_lengths(chd_engine* e, cudaStream_t s, DeltaLengths* out);
// the mode and call-order rules (chd_table.cu, numbered as in DESIGN.md §5): CHD_OK, or the error set and CHD_ERR_STATE (6: or CHD_ERR_INVALID)
chd_status chd_rule_not_table(chd_engine* e, const char* fn);
chd_status chd_rule_table_on_slab(chd_engine* e, const char* fn);
chd_status chd_rule_table(chd_engine* e, const char* fn);
chd_status chd_rule_index_delta(chd_engine* e);
chd_status chd_rule_id_delta(chd_engine* e, uint32_t id_space);
chd_status chd_delta_check(chd_engine* e, bool will_build);
chd_status chd_rule_halo_import(chd_engine* e);
chd_status chd_rule_follow(chd_engine* e, const char* fn);
chd_status chd_rule_no_followers(chd_engine* e, const char* fn);
chd_status chd_rule_no_generated_batch(chd_engine* e, const char* fn);
chd_status chd_rule_one_batch(chd_engine* e, const char* fn);
chd_status chd_rule_merged_batch(chd_engine* e, bool adopted);
chd_status chd_rule_batch_waiting(chd_engine* e, const char* fn, bool generated);
chd_status chd_rule_explicit_subs(chd_engine* e, const char* fn);
chd_status chd_rule_explicit_subs_slab(chd_engine* e, const char* fn);
chd_status chd_rule_facing(chd_engine* e, const char* fn);
chd_status chd_rule_ring_limits(chd_engine* e, const char* fn);
chd_status chd_rule_rings_staged(chd_engine* e, const char* fn);
chd_status chd_rule_no_chain(chd_engine* e, const char* fn, bool fanout_only);
chd_status chd_rule_ring_bytes_reserve(chd_engine* e);
chd_status chd_rule_ring_append(chd_engine* e, bool bytes);
chd_status chd_rule_assemble_rings(chd_engine* e);
chd_status chd_rule_payload_entries(chd_engine* e, uint32_t n_entries);
// followers (chd_follow.cu): the listed slots (n == 0 with slot == nullptr: every slot) follow nothing from now on; d_slot: the
// same list on the device if the caller uploaded it already
chd_status chd_follow_drop(chd_engine* e, const uint32_t* slot, const uint32_t* d_slot, uint32_t n);
// entity-table mode (chd_table.cu): the pass after every table-mode build into copy-input set `c` (sorted ids, handover list
// in ids); the delta's translation to ids, inside its stage; a decoded summary's last successful delta
chd_status chd_table_after_build(chd_engine* e, cudaStream_t s, const CopySet& c);
chd_status chd_table_delta_ids(chd_engine* e, cudaStream_t s);
void chd_table_observe(chd_engine* e, uint32_t delta_build);
}

// The visible delta overflowed: a list outgrew its capacity (CHD_OVF_DELTA) or an id-mode delta met a bad id (CHD_OVF_DELTA_IDS).
// Its lists are not complete, and no read-back copies them.
__host__ __device__ inline bool chd_delta_overflowed(uint64_t n_entered, uint64_t n_left, uint64_t enter_cap, uint64_t leave_cap, bool bad_ids) {
    return n_entered > enter_cap || n_left > leave_cap || bad_ids;
}

// The copy-input set the readers use: the one the last successful build adopted.
static inline const CopySet& chd_copy_in(const chd_engine* e) { return e->copy_set[e->pf_copy.cur]; }

// What set c's sorted_entity, the visible lists and the read-back report: entity indices, or ids in entity-table mode.  The
// slot-valued sorted_ent stays what the delta reads.
static inline const uint32_t* chd_sorted_out(const chd_engine* e, const CopySet& c) { return e->tbl.on ? c.sorted_id : c.sorted_ent; }

// The front position pair: what the set calls and the table-mode kernels write.
static inline const PosSet& chd_pos_front(const chd_engine* e) { return e->pos[e->pf_pos.cur]; }

// The positions the kernels read: the caller's arrays a set call reads in place, else the front pair.  chd_note_pos_read records
// (outside any graph capture) a kernel's read of the front pair, so that a prefetch into it is ordered after that read.
static inline Positions chd_positions(const chd_engine* e) { return e->in_place.x ? e->in_place : Positions{chd_pos_front(e).x, chd_pos_front(e).z}; }
static inline chd_status chd_note_pos_read(chd_engine* e, cudaStream_t s) { return chd_pf_note_read(e, e->pf_pos, e->in_place.x ? -1 : e->pf_pos.cur, s); }

// The ids build positions carry: entity-table slots by the table and the halo after them by d_gid, else d_gid or the index.
static inline EntityIds chd_entity_ids(const chd_engine* e) {
    return e->tbl.on ? EntityIds{e->tbl.d_id_of_slot, e->d_gid, e->n_own} : EntityIds{nullptr, e->have_gid ? e->d_gid : nullptr, 0};
}

// Grow-on-demand buffer: when `need` elements exceed `*cap`, the buffer is replaced (contents not kept) by one of `count`
// elements, the caller's growth policy.  *cap is 0 exactly when there is no buffer.
template <typename T>
static bool ensure_cap(chd_engine* e, T** p, uint64_t* cap, uint64_t need, uint64_t count) {
    if (need <= *cap) return true;
    chd_dfree(e, *p);
    *p = nullptr;
    *cap = 0;
    if (!dalloc(e, p, count)) return false;
    *cap = count;
    return true;
}

static inline unsigned blocks_for(uint64_t n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }

static inline uint64_t mix_key(uint64_t h, uint64_t v) {
    h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    return h;
}
static inline uint64_t key_word(uint64_t v) { return v; }
static inline uint64_t key_word(const void* p) { return (uint64_t)(uintptr_t)p; }

// A graph key: `tag` with each value mixed in turn (a pointer as its address).
template <typename... V>
static inline uint64_t stage_key(uint64_t tag, V... v) {
    uint64_t h = tag;
    ((h = mix_key(h, key_word(v))), ...);
    return h;
}

// Runs `enqueue` (kernel launches + memsets on `s` only, no host sync) either directly or as a CUDA graph replayed on `s`.
// The key is a graph's only identity (it covers every pointer and size the launches bake in): each call site keeps up to 8
// keys in its GraphSet, captures a key at its second sighting and replays it from then on, and gives a key it does not hold
// the least recently used slot and direct launches, so a shape that changes every tick runs direct launches.
template <typename F>
static chd_status run_stage(chd_engine* e, cudaStream_t s, chd_engine::GraphSet& set, uint64_t key, F&& enqueue) {
    key |= 1;  // never 0
    if (!e->use_graphs || s == nullptr) return enqueue();
    chd_engine::GraphSlot* slot = &set.slot[0];  // the slot holding this key, else the least recently used one
    for (chd_engine::GraphSlot& g : set.slot)
        if (g.key == key || (slot->key != key && g.used < slot->used)) slot = &g;
    slot->used = ++set.clock;
    if (slot->key != key) {  // first sighting: run direct, capture next time
        slot->release();
        slot->key = key;
        return enqueue();
    }
    if (slot->exec) {
        CU(e, cudaGraphLaunch(slot->exec, s));
        e->n_launch += slot->nodes;
        e->graph_launches++;
        return CHD_OK;
    }
    const uint64_t l0 = e->n_launch;
    // Stateless entry points (chd_cell_of, chd_query_channel_ids) may be called from other threads and launch into the engine
    // stream: they hold the engine mutex for their whole call, so taking it here keeps their work out of the capture.
    std::lock_guard<std::recursive_mutex> capture_lock(e->mu);
    CU(e, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    chd_status st = enqueue();
    cudaGraph_t g = nullptr;
    cudaError_t r = cudaStreamEndCapture(s, &g);
    if (st != CHD_OK || r != cudaSuccess || !g) {
        if (g) cudaGraphDestroy(g);
        if (st == CHD_OK) {
            e->fail("graph capture failed: %s", cudaGetErrorString(r));
            st = CHD_ERR_CUDA;
        }
        e->use_graphs = false;  // fall back to direct launches for the rest of this engine's life
        cudaGetLastError();
        e->n_launch = l0;
        return st == CHD_OK ? enqueue() : st;
    }
    r = cudaGraphInstantiate(&slot->exec, g, 0);
    cudaGraphDestroy(g);
    if (r != cudaSuccess) {
        slot->exec = nullptr;
        e->use_graphs = false;
        cudaGetLastError();
        e->n_launch = l0;
        return enqueue();
    }
    slot->nodes = e->n_launch - l0;
    e->n_launch = l0;
    e->graph_captures++;
    CU(e, cudaGraphLaunch(slot->exec, s));
    e->n_launch += slot->nodes;
    e->graph_launches++;
    return CHD_OK;
}
