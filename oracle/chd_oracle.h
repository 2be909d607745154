/*
 * chd_oracle.h — CPU ORACLE for the channeld spatial hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This is a plain C++17 restatement (C ABI) of the reference's Go algorithm for
 *   pkg/channeld/spatial.go        (StaticGrid2DSpatialController)
 *   pkg/channeld/message_spatial.go (damping table + interest diff)
 *   pkg/channeld/data.go           (OnUpdate ring + tickData fan-out windows)
 *   pkg/channeld/subscription.go   (fan-out state initialisation)
 *   pkg/channeld/message.go:188-239 (ADJACENT_CHANNELS broadcast recipients)
 *   pkg/common/common.go           (Dist2D / Dot2D / Normalize2D)
 * of channeldorg/channeld @ 61fa8add.  Every function cites the file:line it follows.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library, and only as the checker / the timed CPU baseline — never as the product path.
 *
 * Parity pin status:
 *   - cell id, sphere/box/cone AOI, adjacency: PINNED by the reference's own KATs
 *     (spatial_test.go TestGetChannelId1/2, TestSphereAOI, TestBoxAOI, TestConeAOI,
 *     TestGetAdjacentChannels) — transcribed in tests/test_oracle_kat.py.
 *   - fan-out windows: PINNED by data_test.go:98-166 (F0,F7,F2,F8,F3; doc/design.md:94-109).
 *     data_test.go:168-197 does not follow from the code as written (SURVEY.md §4) and is not used.
 *   - math.Cos (Go stdlib, go 1.25 per go.mod:3; source NOT in the reference tree): restated
 *     from the published Cephes-derived algorithm; cone AOI is "parity unpinned" beyond TestConeAOI.
 *   - SpotsAOI, dist values, damping, interest diff, visible-entity sets, the ADJACENT_CHANNELS broadcast
 *     branch (message.go:188-239): no reference test exists ("parity unpinned" by the reference); the
 *     restatement itself is the ground truth.
 *
 * Numerics: IEEE binary64, round-to-nearest, compiled with -ffp-contract=off (Go/amd64 does not fuse).
 */
#ifndef CHD_ORACLE_H
#define CHD_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* spatial.go:89-124 (fields used by the 2-D grid) + settings.go:94 (SpatialChannelIdStart) */
typedef struct orc_grid {
    double   world_offset_x, world_offset_z;
    double   grid_width, grid_height;
    uint32_t grid_cols, grid_rows;
    uint32_t server_cols, server_rows;
    uint32_t server_interest_border_size;
    uint32_t channel_id_start; /* 0x10000 */
} orc_grid;

enum { ORC_AOI_SPOTS = 1, ORC_AOI_BOX = 2, ORC_AOI_SPHERE = 4, ORC_AOI_CONE = 8 };

/* channeld.proto:436-469 SpatialInterestQuery, flattened (Y is carried by the wire type but unused
 * by the 2-D grid: spatial.go:205,237,272). */
typedef struct orc_query {
    uint32_t kind_mask;
    uint32_t n_spots, n_spot_dists;
    const double*   spot_x;
    const double*   spot_z;
    const uint32_t* spot_dist;
    double box_cx, box_cz, box_ex, box_ez;
    double sph_cx, sph_cz, sph_r;
    double cone_cx, cone_cz, cone_dx, cone_dz, cone_angle, cone_r;
} orc_query;

enum {
    ORC_OK = 0,
    ORC_ERR_OUT_OF_WORLD = 1, /* spatial.go:171-177 / :228-231,:263-266,:309-312 */
    ORC_ERR_BAD_STEP = 2,     /* spatial.go:208-215,:240-247,:277-284 */
    ORC_ERR_NIL = 3,          /* spatial.go:183-185 */
    ORC_ERR_CAPACITY = 4,
    ORC_ERR_ITER_BOUND = 5,   /* guard against the absorbed-step infinite loop / walks of > 2^24 samples (same rule in the CUDA path) */
    ORC_ERR_ANGLE_RANGE = 6   /* |cone angle| >= 2^29 (Go: Payne-Hanek reduction, not restated); same rule in the CUDA path */
};

/* spatial.go:134-139 */
double orc_grid_size(const orc_grid* g);
/* Go's math.Cos as used at spatial.go:295 */
double orc_go_cos(double x);

/* spatial.go:161-180.  Returns ORC_OK and *out_id, or ORC_ERR_OUT_OF_WORLD (and *out_id = 0). */
int orc_get_channel_id(const orc_grid* g, double x, double z, uint32_t* out_id);
/* batch form; out[i] = channel id or 0 on error */
void orc_cell_of(const orc_grid* g, const double* x, const double* z, uint32_t n, uint32_t* out);

/* spatial.go:182-317.  Output sorted by channel id ascending (Go's map order is random; parity
 * is on the key set + dist values).  Returns status; *out_n = number of entries. */
int orc_query_channel_ids(const orc_grid* g, const orc_query* q, uint32_t* out_ids, uint32_t* out_dists,
                          uint32_t cap, uint32_t* out_n);

/* spatial.go:358-381; order as the reference emits (row-major y,x).  Returns count (<=8). */
uint32_t orc_get_adjacent_channels(const orc_grid* g, uint32_t channel_id, uint32_t* out8);

/* message.go:188-239 — recipients of a BroadcastType_ADJACENT_CHANNELS message sent to spatial channel `channel_id`.
 * Every spatial channel's subscribedConnections is given as a CSR by cell index: cell_off[cells+1], conn_id[], conn_type[]
 * (channeldpb.ConnectionType: 1 server, 2 client).  `broadcast` is the BroadcastType mask of the message.
 * Literal restatement: GetAdjacentChannels, append the centre unless ALL_BUT_OWNER, merge all connections of those
 * channels into one map, then the four filters in the reference's order.  out_conn = recipients' connection ids,
 * sorted ascending (the reference iterates a Go map: only the SET is defined).  Returns the count. */
uint32_t orc_adjacent_broadcast(const orc_grid* g, uint32_t channel_id, uint32_t broadcast, uint32_t sender_conn_id,
                                uint32_t client_conn_id, const uint32_t* cell_off, const uint32_t* conn_id,
                                const uint8_t* conn_type, uint32_t* out_conn, uint32_t cap);

/* spatial.go:319-356.  Arrays sized cols*rows. min/max hold x,z (Y is the constant MinY/MaxY). */
void orc_get_regions(const orc_grid* g, double* min_x, double* min_z, double* max_x, double* max_z,
                     uint32_t* channel_id, uint32_t* server_index);

/* message_spatial.go:16-38,65-80: dist -> FanOutIntervalMs; `default_ms` is the SPATIAL channel
 * type's DefaultFanOutIntervalMs used when no damping row matches. */
uint32_t orc_damping_interval_ms(uint32_t dist, uint32_t default_ms);

/* message_spatial.go:82-128 + util.go:105-113 + subscription.go:44-57.
 * existing / wanted are channel-id sets (any order).  Outputs sorted ascending:
 *   unsub = existing \ wanted;  sub_new = wanted \ existing;  kept = wanted ∩ existing. */
void orc_interest_diff(const uint32_t* existing, uint32_t n_existing, const uint32_t* wanted, uint32_t n_wanted,
                       uint32_t* unsub, uint32_t* n_unsub, uint32_t* sub_new, uint32_t* n_sub_new,
                       uint32_t* kept, uint32_t* n_kept);

/* ---- fan-out: literal emulation of one channel's tickData (data.go:149-291, subscription.go:34-102) ---- */
typedef struct orc_channel orc_channel;
typedef struct orc_send {
    uint32_t conn_id;
    uint32_t kind;         /* 0 = FULL (data.go:219-224), 1 = UPDATE (data.go:262-264) */
    uint32_t n_selected;   /* UPDATE: number of merged ring entries */
    uint32_t first_sel;    /* ring position (insertion order, 0-based at time of tick) of first / last selected */
    uint32_t last_sel;
    uint64_t sel_hash;     /* sum of selected messageIndex values mod 2^64 */
    uint64_t last_message_index; /* foc.lastMessageIndex after this step */
    int64_t  window_hi;    /* nextFanOutTime of this step */
} orc_send;

orc_channel* orc_channel_new(void);
void orc_channel_free(orc_channel*);
/* subscription.go:59-87.  now = ch.GetTime() at subscribe. PushFront into the fan-out queue.
 * Returns 0 if newly subscribed, 1 if it already existed (options merged: interval replaced). */
int orc_channel_subscribe(orc_channel*, uint32_t conn_id, int64_t now_ns, uint32_t interval_ms, int32_t delay_ms,
                          int skip_self, int skip_first);
int orc_channel_unsubscribe(orc_channel*, uint32_t conn_id);
/* data.go:149-173 (the merge itself is opaque payload work, not modelled) */
void orc_channel_on_update(orc_channel*, int64_t arrival_ns, uint32_t sender_conn_id);
uint32_t orc_channel_ring_len(const orc_channel*);
/* data.go:175-291.  Appends sends in the order the reference would issue them. Returns count, or
 * (uint32_t)-1 when `cap` is too small or the iteration bound trips (FanOutIntervalMs == 0). */
uint32_t orc_channel_tick_data(orc_channel*, int64_t t_ns, orc_send* out, uint32_t cap);
/* The same tick, additionally reporting for send i: window_lo[i] = the connection's lastFanOutTime when the step began
 * (data.go:205,226), self_skipped[i] = how many of the connection's own buffered updates fell into the window and were
 * left out by SkipSelfUpdateFanOut (data.go:239-242), and the ring positions merged into its payload as a CSR
 * (sel_off[n+1], sel_pos[]) — the exact payload identity used to check the window classes (SURVEY.md §8f rank 1).
 * Returns (uint32_t)-1 when cap / sel_cap are too small. */
uint32_t orc_channel_tick_data_ex(orc_channel*, int64_t t_ns, orc_send* out, uint32_t cap, int64_t* window_lo, uint32_t* self_skipped,
                                  uint32_t* sel_off, uint32_t* sel_pos, uint32_t sel_cap);
/* read back per-connection state: returns 0 if found */
int orc_channel_get_state(const orc_channel*, uint32_t conn_id, int64_t* last_fanout, int* had_first,
                          uint64_t* last_msg_index);

/* ---- derived: per-subscriber visible-entity lists (SURVEY.md §8 a14) ----
 * visible(s) = { e : cell(pos_e) in keys(QueryChannelIds(query_s)) }, canonical order (cell asc, entity idx asc).
 * Sphere-only batch (the benchmark shape).  pair_off[nq+1], vis_off[nq+1] (u64).  status[nq].
 * Buffers may be NULL to only count.  Returns 0 or ORC_ERR_CAPACITY. n_threads>=1. */
int orc_sphere_tick(const orc_grid* g, const double* ex, const double* ez, uint32_t n_ent,
                    const double* cx, const double* cz, const double* r, uint32_t nq,
                    uint32_t* status, uint64_t* pair_off, uint32_t* pair_cell, uint32_t* pair_dist, uint64_t pair_cap,
                    uint64_t* vis_off, uint32_t* vis_entity, uint64_t vis_cap, int n_threads);

/* Timed CPU baseline: for queries [q_begin,q_end) run the per-query map-building QueryChannelIds and
 * copy every visible entity index into a per-thread scratch list (the work the reference's fan-out
 * implies), using cell lists built from all n_ent entities (build != 0: rebuilt inside the call, in parallel over n_threads;
 * build == 2: rebuilt serially, the round-1 behaviour, kept for comparison).  Threads come from a persistent pool.
 * Returns a checksum (sum of visible counts + pair counts) so the work cannot be optimised away. */
uint64_t orc_baseline_run(const orc_grid* g, const double* ex, const double* ez, uint32_t n_ent,
                          const double* cx, const double* cz, const double* r, uint32_t q_begin, uint32_t q_end,
                          int n_threads, int build);

#ifdef __cplusplus
}
#endif
#endif
