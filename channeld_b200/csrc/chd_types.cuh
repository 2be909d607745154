// chd_types.cuh — plain structs shared between the kernels (csrc/*.cuh) and the host-side launch code (csrc/*.cu).
#pragma once
#include "chd_device.cuh"

namespace chd {

// tile geometry the host-side sizing code shares with the kernels
constexpr int BUILD_THREADS = 256;
constexpr int BUILD_WARPS = BUILD_THREADS / 32;
constexpr int BUILD_ROUNDS = 8;
constexpr int BUILD_TILE = BUILD_THREADS * BUILD_ROUNDS;  // 2048 entities per tile
constexpr int BUILD_MAX_BINS = 1024;
constexpr int EMIT_THREADS = 256;
// Two rows (an 8 KB tile) of the two-segment emit kernel.  Measured on an H100 SXM (80 GB HBM3, 400 W power limit), benchmark
// config, emit kernel per tick, when it still read the four phase copies: 0.858 ms with 2 rows and 8 CTAs per SM, 0.875 ms with 4
// rows and 6 CTAs (40 registers), 1.53 ms with 4 rows and 8 CTAs (32 registers, 72 bytes spilled per thread), 1.29 ms with 8
// rows and 3 CTAs.  Reading phase copy 0 alone (shuffles between lanes) needs 40 registers: 8 CTAs per SM (32 registers) spill
// 44 bytes per thread and took 0.851 ms, 6 CTAs per SM took 0.641 ms (H100 SXM, 700 W, the kernel alone at the benchmark shape).
#ifndef CHD_EMIT_ROWS
#define CHD_EMIT_ROWS 2
#endif
#ifndef CHD_EMIT_MIN_BLOCKS
#define CHD_EMIT_MIN_BLOCKS 6
#endif
// Dynamic shared memory the two-segment emit kernel asks for WITHOUT using it: 0 lets as many CTAs as the register file allows
// be emit CTAs; a larger value caps them per SM, to keep slots free for the latency-bound kernels of the second stream.
#ifndef CHD_EMIT_DYN_SMEM
#define CHD_EMIT_DYN_SMEM 0
#endif
// Tiles one CTA of the two-segment emit kernel copies, one after the other (tiles b, b + grid, ...); the next descriptor is
// prefetched into L1 while the current tile is copied.  Measured on an H100 SXM (80 GB HBM3, 700 W power limit), benchmark
// config, emit kernel per tick: 0.718-0.720 ms with 1 tile per CTA, 0.679 ms with 2, 0.682-0.683 ms with 4, 0.694 ms with 8,
// 0.712 ms with 16; 2 tiles without the prefetch: 0.682 ms (DESIGN §8).
#ifndef CHD_EMIT_TILES_PER_CTA
#define CHD_EMIT_TILES_PER_CTA 2
#endif
constexpr int EMIT_TILES_PER_CTA = CHD_EMIT_TILES_PER_CTA;
constexpr int EMIT_ROWS = CHD_EMIT_ROWS;                    // 16-byte chunks per thread per tile
constexpr int EMIT_TILE = EMIT_THREADS * 4 * EMIT_ROWS;     // 2048 entries = 8 KB of output per tile
constexpr int EMIT_SMEM_PAIRS = 256;                        // pairs per tile staged in shared memory (one per thread)
// the general (warp-tile) kernel: 8 x 16 bytes per lane = 4 KB of output per warp tile
constexpr int EMIT_WARP_WARPS = EMIT_THREADS / 32;
constexpr int EMIT_WARP_CHUNKS = 8;
constexpr int EMIT_WARP_TILE = 32 * EMIT_WARP_CHUNKS * 4;   // 1024 entries
constexpr int EMIT_WARP_SMEM_PAIRS = 64;

// Per-tile copy descriptor written by the partition pass: the emit kernel needs ONE 16-byte load (broadcast to the CTA)
// before it can issue its data loads, instead of a chain of three dependent index loads (first pair -> offsets / cell ->
// cell start).  A tile is "simple" if at most two pairs' lists intersect it (always the case when cells hold more entities
// than a tile: 4 444 vs 4 096 on the benchmark config); other tiles take the general path (segment table in shared memory).
struct TileDesc {
    uint32_t src0;  // base of the first segment in the sorted entity array: slot o of the tile <- sorted[src0 + o]
    uint32_t src1;  // the same for the second segment (slots o >= end0; stored minus end0, may wrap below zero)
    uint32_t ends;  // end0 | end1 << 16 (relative to the tile base, <= EMIT_TILE); bit 31 = not simple
    uint32_t p0;    // the pair that owns the tile's first slot (general path)
};
static_assert(EMIT_TILE <= 0x7FFF, "segment ends are packed into 15 bits");

struct QueryDev {
    uint32_t n;
    const uint32_t* sub;
    const uint8_t* kind;
    const double *sph_cx, *sph_cz, *sph_r;
    const double *box_cx, *box_cz, *box_ex, *box_ez;
    const double *cone_cx, *cone_cz, *cone_dx, *cone_dz, *cone_angle, *cone_r;
    const uint32_t *spot_off, *spot_ndist;
    const double *spot_x, *spot_z;
    const uint32_t* spot_dist;
    // nullptr except in a merged batch (chd_follow_queries_with): [n], entry i names a kind whose arrays the host part lacked
    const uint8_t* missing;
};

// (query_kernel, and follow_merge_kernel for a merged batch's host part)
__device__ __forceinline__ uint32_t query_kind(const QueryDev& q, uint32_t i) { return q.kind ? q.kind[i] : (uint32_t)CHD_AOI_SPHERE; }

// A kind bit whose arrays the batch does not supply (CHD_Q_ERR_MISSING_ARRAY).  Spots without spot_off are ignored, not missing.
__device__ __forceinline__ bool query_arrays_missing(const QueryDev& q, uint32_t kind) {
    return ((kind & CHD_AOI_BOX) && (!q.box_cx || !q.box_cz || !q.box_ex || !q.box_ez)) ||
           ((kind & CHD_AOI_SPHERE) && (!q.sph_cx || !q.sph_cz || !q.sph_r)) ||
           ((kind & CHD_AOI_CONE) && (!q.cone_cx || !q.cone_cz || !q.cone_dx || !q.cone_dz || !q.cone_angle || !q.cone_r)) ||
           ((kind & CHD_AOI_SPOTS) && q.spot_off && (!q.spot_x || !q.spot_z || !q.spot_dist));
}

struct Bbox {
    uint32_t gx0, gy0, bw, bh;  // bw == 0 => empty
};

struct PairBuf {
    uint32_t* off;         // [S+1]
    uint32_t* sub;         // [P] owning subscriber slot
    uint32_t* cell;        // [P] cell index
    uint32_t* dist;        // [P]
    uint32_t* interval;    // [P] FanOutIntervalMs
    uint8_t* flags;        // [P]
    int64_t* last;         // [P] lastFanOutTime (ns)
    uint64_t* last_index;  // [P] lastMessageIndex
};
enum : uint8_t { PF_HAD_FIRST = 1, PF_NEW = 2, PF_SKIP_SELF = 4 };

struct Counters {  // device mirror of chd_tick_summary's counters
    unsigned long long n_pairs, n_visible;
    uint32_t n_entities_in_world, n_query_errors, n_sub_new, n_unsub, n_kept, n_due, n_handover, overflow;
    unsigned long long required_pairs, required_window_cells, required_visible;
    uint32_t required_due;
    uint32_t delta_build;  // entity-table mode: the build number the last successful visible delta measured (chd_table.cuh)
};

// Pending lifecycle change of a subscriber slot, applied by the next interest update (chd_interest.cuh):
enum : uint8_t {
    SLOT_NORMAL = 0,
    SLOT_REMOVE = 1,  // chd_remove_subscribers: every subscription of the slot is reported as unsubscribed, the slot is freed
    SLOT_DROP = 2,    // chd_migrate_out: the slot's state was packed for another rank; its run vanishes without unsub entries
    SLOT_IMPORT = 3   // chd_migrate_in: the slot's previous run comes out of the gathered migration blob (MigView)
};

// Subscriber state in flight between ranks: every rank contributes one fixed-size blob to the tick's all-gather (after its
// border records).  Word layout of a blob (u32 words; Ms = max_subs, Mp = max_pairs, both even):
//   [0] n_sub  [1] n_pairs  [2..3] pad | off[Ms+2] | conn[Ms] | cell[Mp] | dist[Mp] | interval[Mp] | flags[Mp] |
//   last[Mp] (i64) | last_index[Mp] (u64)
struct MigView {
    const uint32_t* base;   // nullptr: no migration data this tick
    uint64_t stride_words;  // distance between the blobs of consecutive ranks
    uint32_t max_subs, max_pairs;
    __host__ __device__ static uint64_t words(uint32_t ms, uint32_t mp) { return 4ull + (ms + 2ull) + ms + 4ull * mp + 4ull * mp; }
    __host__ __device__ uint64_t o_off() const { return 4; }
    __host__ __device__ uint64_t o_conn() const { return o_off() + max_subs + 2ull; }
    __host__ __device__ uint64_t o_cell() const { return o_conn() + max_subs; }
    __host__ __device__ uint64_t o_dist() const { return o_cell() + max_pairs; }
    __host__ __device__ uint64_t o_interval() const { return o_dist() + max_pairs; }
    __host__ __device__ uint64_t o_flags() const { return o_interval() + max_pairs; }
    __host__ __device__ uint64_t o_last() const { return o_flags() + max_pairs; }
    __host__ __device__ uint64_t o_lidx() const { return o_last() + 2ull * max_pairs; }
};

struct DiffOut {  // the two interest-diff lists of a tick: (subscriber slot, channel id)
    uint32_t *new_sub, *new_ch, *gone_sub, *gone_ch;
};

struct RingDev {
    const uint32_t* off;        // ring of cell c = entries [off[c], end[c]): host-owned rings are a CSR (end = off + 1),
    const uint32_t* end;        // device-owned rings (chd_rings_init) keep begin / end cursors per cell
    const int64_t* arrival;     // insertion order per cell
    const uint32_t* sender;
    const uint64_t* index;
    const uint64_t* channel_msg_index;  // [C] or nullptr
    const uint32_t* total;              // entries uploaded (device scalar): offsets are clamped to it
    const int64_t* start;               // [C] ChannelTime origin of each channel (channel.go:28-37,178) or nullptr = one shared origin
};

// Payload identity of a decision (window classes, chd_classes.cuh): two decisions of one channel carry the same merged
// payload if they are both FULL, or if they start from the same lastFanOutTime (`lo`), end at the same nextFanOutTime
// (the record's window_hi) and neither subscriber had an own update left out of that window; a decision with
// self-skipped updates is its own class.  word = cell << 34 | kind << 33 | skipped << 32 | (skipped ? subscriber slot : 0).
struct DueKey {
    int64_t lo;
    uint64_t word;
};

struct HandoverOut {
    uint32_t* entity;
    uint32_t* src_cell;
    uint32_t* dst_cell;
    uint32_t* count;  // device counter (may exceed cap: required size)
    uint32_t cap;
};

// The cell CSR a sort by cell publishes (chd_cell_sort).  A single-pass sort (digit == key) publishes it straight from the
// scanned histogram (cell_start[c] = #keys < c, load_base): fused into the scatter when cell_start != null, or by
// publish_cell_start_kernel in a split build, replacing a separate boundaries kernel
struct ScatterExtras {
    uint32_t* cell_start;
    uint32_t cells;
    uint32_t* n_in_world;
};

// The id build position p carries (chd_entity_ids): below `own` an entity-table slot's, else gid's (global ids, and the halo ids
// the import writes) or p without gid.  Halo ids never enter own_ids: a later spawn into such a position must not inherit one.
struct EntityIds {
    const uint32_t *__restrict__ own_ids, *__restrict__ gid;
    uint32_t own;
    __device__ __forceinline__ uint32_t at(uint32_t p) const { return p < own ? own_ids[p] : (gid ? gid[p] : p); }
};

// ---- the entity table's id -> slot words and their lookup (layout: chd_table.cuh), shared with the followers' entity lookup
constexpr uint64_t TBL_EMPTY = 0;
constexpr uint64_t TBL_TOMB = 0xFFFFFFFFull << 32;
constexpr uint32_t TBL_NONE = 0xFFFFFFFFu;

__host__ __device__ __forceinline__ uint64_t tbl_home(uint32_t id, uint32_t bits) { return ((uint64_t)id * 0x9E3779B97F4A7C15ull) >> (64 - bits); }

__device__ __forceinline__ uint32_t tbl_find(const uint64_t* __restrict__ table, uint32_t bits, uint32_t id, uint64_t* where) {
    const uint64_t mask = (1ull << bits) - 1ull;
    if (id == 0u || id == TBL_NONE) return TBL_NONE;
    for (uint64_t h = tbl_home(id, bits);; h = (h + 1) & mask) {
        const uint64_t w = table[h];
        if (w == TBL_EMPTY) return TBL_NONE;
        if ((uint32_t)(w >> 32) == id) {
            if (where) *where = h;
            return (uint32_t)w;
        }
    }
}

// ---- followers (chd_follow.cuh)
// Per-slot binding state, [max_subscribers] each.  kind == 0: the slot follows nothing.
struct FollowDev {
    uint32_t* entity;  // entity index, or table id in entity-table mode
    uint8_t* kind;     // CHD_AOI_SPHERE | BOX | CONE mask
    double *sph_r, *box_ex, *box_ez, *cone_dx, *cone_dz, *cone_angle, *cone_r;
    double *last_x, *last_z;  // centre of the last query generated for the slot
    uint8_t* dirty;           // bound or re-bound since the last batch that selected the slot, or its entity was missing then
    uint32_t* tslot;          // entity-table mode: the table slot the id was last found in (validated against slot -> id on use)
    uint32_t* res;            // what the last generation did with the slot: batch entry, or FOLLOW_NO_QUERY | reason
    uint8_t* ovr;             // a host entry of the merged batch names the slot (set by follow_merge_kernel, cleared by FollowFlag)
};

// Frames of followers (chd_follow_set_frame, include/chd_gpu_facing.h), [max_subscribers] each, allocated by the first frame.
// on == 0: the slot's follower is plain.
struct FollowFrame {
    uint8_t* on;
    double *off_fwd, *off_right, *rot_cos, *rot_sin;
    double *last_fx, *last_fz;  // the facing the last query was generated from (0, 0: none)
    double *cx, *cz, *dx, *dz;  // that query's centre and cone direction (chd_get_follow_frame)
};

// The generated batch: a query batch's SoA in device memory.  The spot arrays and `missing` are used by merged batches only.
struct FollowBatch {
    uint32_t* sub;
    uint8_t* kind;
    double *sph_cx, *sph_cz, *sph_r, *box_cx, *box_cz, *box_ex, *box_ez, *cone_cx, *cone_cz, *cone_dx, *cone_dz, *cone_angle, *cone_r;
    uint32_t* n_selected;
    uint32_t *spot_off, *spot_ndist;  // [Q + 1], [Q]
    double *spot_x, *spot_z;          // [spot capacity], grown on demand
    uint32_t* spot_dist;
    uint8_t* missing;                 // [Q]
};

struct BcastDev {
    uint32_t n;
    const uint32_t *channel, *flags, *sender, *client;
};

}  // namespace chd
