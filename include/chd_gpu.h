/*
 * chd_gpu.h — C ABI of the H100-native spatial interest-management + fan-out engine (libchd_b200.so).
 *
 * This is the drop-in boundary behind channeld's SpatialController plugin surface
 * (reference: channeldorg/channeld @ 61fa8add, pkg/channeld/spatial.go:17-35).  A cgo shim binds exactly
 * these entry points (INTEGRATION.md, go/gpucontroller.go).  Plain pointers and sizes only; no C++/torch
 * types; integer status codes; no exceptions cross the ABI.  Pointer retention: the synchronous entry points (chd_cell_of,
 * chd_query_channel_ids, chd_adjacent_broadcast, chd_get_*, chd_fetch_results, chd_summary) are done with every caller pointer
 * when they return; the stream-ordered ones (chd_set_*, chd_prefetch_*, chd_tick, chd_update_interest with HOST arrays) read
 * caller memory asynchronously until the next synchronising call — such buffers must be C memory (chd_alloc_pinned), never
 * Go-managed memory (cgo pointer rules, INTEGRATION.md).  Pointer arguments may be host (pageable or pinned) or device pointers unless
 * stated otherwise.  HOST inputs are copied (cudaMemcpyAsync on the engine's stream; pinned memory makes that
 * asynchronous) and may be reused once the call that consumes them has been followed by chd_summary / chd_sync /
 * a chd_get_* call.  DEVICE inputs of the tick path (chd_set_entities, chd_set_rings, the arrays of a
 * chd_query_batch) that live on the engine's GPU are consumed IN PLACE (zero copy): the producer keeps them valid
 * and unmodified until the tick that reads them has finished.
 *
 * Threading: one tick driver per engine handle (thread-compatible).  chd_cell_of / chd_query_channel_ids
 * take an internal mutex and may be called from any thread (the reference calls GetChannelId /
 * QueryChannelIds concurrently from channel goroutines, spatial.go:20-29).
 *
 * There is NO CPU fallback: every compute entry point runs sm_90a kernels and returns CHD_ERR_CUDA if no
 * device is usable.
 */
#ifndef CHD_GPU_H
#define CHD_GPU_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define CHD_ABI_VERSION 1

typedef struct chd_engine chd_engine;

typedef enum chd_status {
    CHD_OK = 0,
    CHD_ERR_INVALID = 1,  /* bad argument / config (LoadConfig validation, spatial.go:146-157) */
    CHD_ERR_CUDA = 2,     /* CUDA runtime failure or no device; see chd_last_error */
    CHD_ERR_CAPACITY = 3, /* an output or scratch capacity in chd_limits was exceeded; summary.required_* says by how much */
    CHD_ERR_STATE = 4     /* call order violated (e.g. emit before build) */
} chd_status;

/* Grid constants.  Replaces StaticGrid2DSpatialController's config fields (spatial.go:89-124, JSON in
 * config/spatial_static_*.json) + GlobalSettings.SpatialChannelIdStart (settings.go:94). */
typedef struct chd_grid_cfg {
    double   world_offset_x, world_offset_z;
    double   grid_width, grid_height;
    uint32_t grid_cols, grid_rows;
    uint32_t server_cols, server_rows;
    uint32_t server_interest_border_size;
    uint32_t channel_id_start; /* 0x10000 */
} chd_grid_cfg;

/* Capacities (device allocations are made once in chd_create; nothing allocates on the tick path). */
typedef struct chd_limits {
    uint32_t max_entities;
    uint32_t max_subscribers;
    uint32_t max_queries;       /* per chd_update_interest / chd_query_channel_ids batch */
    uint32_t max_spots;         /* total SpotsAOI spots per batch */
    uint64_t max_pairs;         /* (subscriber, cell) subscriptions alive at once */
    uint64_t max_window_cells;  /* query scratch: sum over the batch of each query's cell bounding box */
    uint64_t max_visible;       /* expanded visible-entity list entries per tick */
    uint32_t max_ring_entries;  /* total update-ring entries over all cells */
    uint32_t max_due;           /* fan-out decisions per tick */
    /* SPATIAL channel-type settings the reference reads from GlobalSettings.ChannelSettings
     * (settings.go:97-103,237-243; subscription.go:21-31): */
    uint32_t default_fanout_interval_ms; /* used when dist matches no damping row (message_spatial.go:68-72) */
    int32_t  default_fanout_delay_ms;
} chd_limits;

/* Fills `lim` with capacities sized for n_entities / n_subscribers (helper; edit before chd_create). */
void chd_default_limits(const chd_grid_cfg* cfg, uint32_t n_entities, uint32_t n_subscribers, chd_limits* lim);

/* Replaces InitSpatialController + LoadConfig (spatial.go:40-74,141-159).  Validates like LoadConfig except
 * that ServerInterestBorderSize == 0 is accepted: the reference discards that error (spatial.go:68) and both
 * benchmark configs rely on it.  `device` = CUDA ordinal. */
chd_status chd_create(const chd_grid_cfg* cfg, const chd_limits* lim, int device, chd_engine** out);
void chd_destroy(chd_engine* e);
/* Last error text of this engine (or of chd_create when e == NULL).  Valid until the next call. */
const char* chd_last_error(const chd_engine* e);
/* Run all work on this cudaStream_t (default: a private non-blocking stream).  torch passes its current stream. */
chd_status chd_set_stream(chd_engine* e, void* cuda_stream);
/* Blocks until all work queued on the engine stream has finished. */
chd_status chd_sync(chd_engine* e);

/* Pinned host memory for the per-tick staging buffers (plain C memory, legal to hold from Go). */
void* chd_alloc_pinned(uint64_t bytes);
/* NUMA node of the GPU (from sysfs; -1 = unknown).  Pinned memory is placed by first touch: run the tick driver (the thread that
 * calls chd_alloc_pinned) on that node's cores and the per-tick uploads cross no socket interconnect. */
int chd_device_numa_node(int device);
void chd_free_pinned(void* p);

/* ---- GetChannelId, batched (spatial.go:161-180; the batch form is handleQuerySpatialChannel,
 * message_spatial.go:335-370).  out_channel_id[i] = channel id, or 0 where the reference returns an error
 * (outside [0,cols) x [0,rows), NaN, +-Inf, huge).  Synchronous. */
chd_status chd_cell_of(chd_engine* e, const double* x, const double* z, uint32_t n, uint32_t* out_channel_id);
/* The same with an explicit validity flag per position (out_valid[i] = 1 / 0; may be NULL): needed when
 * channel_id_start == 0, where channel id 0 is a real cell and cannot double as the error value. */
chd_status chd_cell_of_valid(chd_engine* e, const double* x, const double* z, uint32_t n, uint32_t* out_channel_id, uint8_t* out_valid);

/* ---- entity positions (SoA).  Replaces the per-cell entity maps the reference keeps in
 * SpatialChannelData.Entities (pkg/unrealpb/extension.go:38-62) fed by AddEntity/RemoveEntity
 * (spatial.go:606-609,702-736).  Entity i has id i (the host maps it to EntityChannelIdStart + i).  Entity-table mode
 * (chd_entity_table_init, below) replaces these snapshots with spawn / move / despawn events keyed by id. */
chd_status chd_set_entities(chd_engine* e, const double* x, const double* z, uint32_t n);
/* Double-buffered upload for pipelined hosts: chd_prefetch_entities starts copying the NEXT tick's host positions
 * into the engine's second pair of position buffers on a dedicated upload stream and returns immediately; it may be
 * called while a tick is in flight (the H2D transfer then overlaps that tick's kernels).  x / z must stay valid until
 * chd_adopt_prefetched has been followed by chd_summary / chd_sync / chd_fetch_results.  chd_adopt_prefetched makes the
 * prefetched positions the current ones (replaces chd_set_entities for that tick; CHD_ERR_STATE if nothing was
 * prefetched).  The second buffer pair is allocated on the first prefetch. */
chd_status chd_prefetch_entities(chd_engine* e, const double* x, const double* z, uint32_t n);
/* The same two calls for positions that ARE floats at the source: channeld's entities move as unrealpb.FVector (three floats,
 * pkg/unrealpb/unreal_common.proto:55-59) and only become SpatialInfo doubles by float64(*vec.X) (pkg/unrealpb/extension.go:10-24;
 * x = FVector.X, z = FVector.Y).  The widening is exact and is done on the device behind the copy, so a snapshot costs 8 instead of
 * 16 bytes per entity on PCIe and every result is bit-identical to chd_set_entities fed with the widened values.  Device-resident
 * float arrays (16-byte aligned) are widened in place of the copy. */
chd_status chd_set_entities_f32(chd_engine* e, const float* x, const float* z, uint32_t n);
chd_status chd_prefetch_entities_f32(chd_engine* e, const float* x, const float* z, uint32_t n);
/* (chd_prefetch_queries / chd_prefetch_rings, declared after chd_set_rings, do the same for the other per-tick inputs.) */
chd_status chd_adopt_prefetched(chd_engine* e);
/* Device pointers of the resident position arrays, for producers that write positions on the GPU. */
chd_status chd_entity_buffers(chd_engine* e, double** d_x, double** d_z, uint32_t* n);

/* Declares that the resident position arrays hold n entities (after writing them through chd_entity_buffers). */
chd_status chd_set_entity_count(chd_engine* e, uint32_t n);

/* GetChannelId for every resident entity (the first half of chd_build; idempotent until positions change).
 * Also runs handover detection against the previous assignment. */
chd_status chd_assign_cells(chd_engine* e);

/* Spatial-hash build: cell id per entity (GetChannelId), stable counting sort into the cell CSR
 * (cell asc, entity id asc), and — when a previous build exists — handover detection, the prefix of
 * Notify (spatial.go:612-626): entities whose cell changed since the previous build. */
chd_status chd_build(chd_engine* e);

/* ---- subscribers: slot s in [0,n) <-> connection id (Connection.Id(), used for SkipSelfUpdateFanOut,
 * data.go:240).  Resets all subscriptions. */
chd_status chd_set_subscribers(chd_engine* e, const uint32_t* conn_id, uint32_t n);

/* ---- subscriber lifecycle: slots are managed by the HOST (it owns the connection table, connection.go).  Neither call
 * disturbs any other slot's subscriptions or fan-out state (lastFanOutTime, hadFirstFanOut, lastMessageIndex).
 *   chd_add_subscribers    slot[i] (free: never used, or removed before) becomes connection conn_id[i]; it has no subscriptions
 *                          until its first query (SubscribeToChannel then starts it like any new pair, subscription.go:60-87)
 *   chd_remove_subscribers UnsubscribeFromChannel for every spatial channel of the slot (subscription.go:104-125; also what
 *                          tickConnections does for a closed connection, channel.go:414-475): applied by the NEXT
 *                          chd_update_interest / chd_tick with a batch (an empty batch will do) — the slot's subscriptions appear
 *                          in that update's unsub list, a query for the slot in the same batch is ignored, the slot is free
 *                          afterwards.
 * slot / conn_id are HOST arrays (copied before the call returns).  Slots may exceed the count given to chd_set_subscribers
 * (up to chd_limits.max_subscribers). */
chd_status chd_add_subscribers(chd_engine* e, const uint32_t* slot, const uint32_t* conn_id, uint32_t n);
chd_status chd_remove_subscribers(chd_engine* e, const uint32_t* slot, uint32_t n);

enum { CHD_AOI_SPOTS = 1, CHD_AOI_BOX = 2, CHD_AOI_SPHERE = 4, CHD_AOI_CONE = 8 };

/* A batch of SpatialInterestQuery (channeld.proto:436-469), SoA.  Arrays of kinds no query uses may be
 * NULL.  Y components are not carried: the 2-D grid never reads them (spatial.go:205,237,272).
 * At most one query per subscriber slot per batch (the host coalesces; the reference would apply them
 * in arrival order and only the last one's subscriptions survive). */
typedef struct chd_query_batch {
    uint32_t        n;
    const uint32_t* sub;   /* [n] subscriber slot (UpdateSpatialInterestMessage.connId -> slot), or NULL = identity (query i is
                              subscriber slot i, n <= subscribers); ignored by chd_query_channel_ids */
    const uint8_t*  kind;  /* [n] CHD_AOI_* mask, or NULL = all CHD_AOI_SPHERE */
    const double *sph_cx, *sph_cz, *sph_r;
    const double *box_cx, *box_cz, *box_ex, *box_ez;
    const double *cone_cx, *cone_cz, *cone_dx, *cone_dz, *cone_angle, *cone_r;
    const uint32_t* spot_off;    /* [n+1] CSR into spot_* (NULL when no query has spots) */
    const uint32_t* spot_ndist;  /* [n] how many leading spots of query i carry an explicit dist (len(Dists)) */
    const double *  spot_x, *spot_z;
    const uint32_t* spot_dist;   /* [spot_off[n]]; 0xFFFFFFFF is reserved */
} chd_query_batch;

/* Per-query status (the reference's error returns, spatial.go:208-215,228-231,...). */
enum {
    CHD_Q_OK = 0,
    CHD_Q_ERR_OUT_OF_WORLD = 1, /* centre of a box/sphere/cone outside the world: (nil, err) */
    CHD_Q_ERR_BAD_STEP = 2,     /* radius / extent <= 0 */
    CHD_Q_ERR_ITER_BOUND = 5,   /* step absorbed by a huge coordinate (v + step == v: the reference would loop forever), or a
                                   lattice walk of more than 2^24 samples (cut off: a documented deviation) */
    CHD_Q_ERR_ANGLE_RANGE = 6,  /* |cone angle| >= 2^29: Go switches to Payne-Hanek reduction, not reproduced */
    CHD_Q_ERR_CAPACITY = 7,     /* the query's cell window did not fit chd_limits.max_window_cells (CHD_OVF_WINDOW is raised):
                                   like every failed query it leaves the subscriber's subscriptions untouched.  Only a query that
                                   needs a window can get it: one whose window is empty (spots only, or shapes that miss the
                                   grid) runs its spots or fails with its own status however full the scratch is */
    CHD_Q_ERR_MISSING_ARRAY = 8 /* a kind bit is set but that kind's arrays were not supplied in the batch */
};

/* ---- QueryChannelIds, batched and stateless (spatial.go:182-317).  CSR output, entries of one query sorted
 * by channel id ascending (the reference returns a Go map: order is unspecified, parity is on keys+dists).
 * out_off[n+1], out_status[n]; out_channel_id/out_dist sized `cap`.  Synchronous. */
chd_status chd_query_channel_ids(chd_engine* e, const chd_query_batch* q, uint32_t* out_status, uint32_t* out_off,
                                 uint32_t* out_channel_id, uint32_t* out_dist, uint64_t cap);

/* ---- handleUpdateSpatialInterest, batched (message_spatial.go:41-129): query -> damping
 * (message_spatial.go:16-38) -> diff against the subscriber's current spatial subscriptions (util.go:105-113)
 * -> SubscribeToChannel / UnsubscribeFromChannel state changes (subscription.go:34-125): new pairs start with
 * lastFanOutTime = now_ns + delay, hadFirstFanOut = false; kept pairs keep their fan-out state and take the
 * new interval; a query that errors leaves that subscriber's subscriptions untouched (message_spatial.go:60-63).
 * Asynchronous (stream-ordered). */
chd_status chd_update_interest(chd_engine* e, const chd_query_batch* q, int64_t now_ns);

/* ---- expanded per-subscriber visible-entity lists: for each subscriber the concatenation, in channel-id
 * order, of the entity lists of its subscribed cells (SURVEY.md §8 a14).  Asynchronous. */
chd_status chd_emit_visible(chd_engine* e);

/* ---- update rings: the per-channel updateMsgBuffer metadata (data.go:46-51) in insertion order, CSR by cell
 * index (channel id - channel_id_start): ring_off[cells+1], n_entries = ring_off[cells].  channel_msg_index[cells] = ChannelData.msgIndex
 * (data.go:25,158) or NULL for zeros.  The host owns OnUpdate/eviction (data.go:149-173): payload merging is
 * opaque protobuf work.  Call order: before chd_begin_interest(..., with_fanout = 1), whose fan-out reads the rings on the
 * engine's second stream until chd_tick joins it; in between it returns CHD_ERR_STATE (with with_fanout = 0 it is accepted). */
chd_status chd_set_rings(chd_engine* e, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival_ns,
                         const uint32_t* sender_conn_id, const uint64_t* message_index, const uint64_t* channel_msg_index);
/* The same for the other per-tick inputs: the query batch (consumed by the next chd_begin_interest / chd_update_interest
 * called with q == NULL) and the update rings (arguments as chd_set_rings; CHD_ERR_STATE on device-owned rings, see
 * chd_rings_init).  Each kind has two staging sets: a prefetch fills the one not adopted last, and only after the work that
 * last read it, so a host that prefetches for tick k+1 while tick k runs alternates between them and never waits for tick k.
 * A second prefetch of one kind before an adoption replaces the first.  chd_adopt_prefetched hands over everything
 * prefetched since the last adoption (any subset of positions / queries / rings). */
chd_status chd_prefetch_queries(chd_engine* e, const chd_query_batch* q);
chd_status chd_prefetch_rings(chd_engine* e, const uint32_t* ring_off, uint32_t n_entries, const int64_t* arrival, const uint32_t* sender,
                              const uint64_t* index, const uint64_t* ch_msg_index);


/* ---- device-owned rings: the buffer half of ChannelData.OnUpdate (data.go:149-173) on the GPU, for every channel at once.
 * chd_rings_init switches the engine from host-owned ring snapshots (chd_set_rings every tick: 20 bytes x every live entry) to rings
 * that live in HBM: capacity_per_cell (> 512) entries per cell, cells x capacity_per_cell <= chd_limits.max_ring_entries.
 * chd_rings_append applies a tick's updates: CSR by cell (upd_off[cells + 1]) in arrival order per cell; for each one
 * msgIndex++, push (arrival, sender, msgIndex), and — if the buffer holds more than 512 entries and its OLDEST is older than the
 * channel's maxFanOutIntervalMs (tracked on the device: it grows when a subscription with a longer interval is created,
 * subscription.go:84-86) — pop that one.  Merging the update into the channel's data message (opaque protobuf) stays with the
 * host.  chd_get_rings reads the live rings back as the CSR chd_set_rings takes (tests, recovery).  Stream-ordered except
 * chd_get_rings.  Offsets past n_updates are read as n_updates.  Call order: chd_rings_init, chd_rings_append and
 * chd_set_channel_start_times go before chd_begin_interest (the interest update and the fan-out it starts read the rings, the
 * start times and maxFanOutIntervalMs) or after the chd_tick that joins it; in between they return CHD_ERR_STATE and change
 * nothing. */
chd_status chd_rings_init(chd_engine* e, uint32_t capacity_per_cell);
chd_status chd_rings_append(chd_engine* e, const uint32_t* upd_off, uint32_t n_updates, const int64_t* arrival_ns, const uint32_t* sender_conn_id);
chd_status chd_get_rings(chd_engine* e, uint32_t* ring_off, int64_t* arrival_ns, uint32_t* sender_conn_id, uint64_t* message_index,
                         uint64_t* channel_msg_index, uint32_t cap_entries);
/* ChannelTime origin per channel (channel.go:28-37,178: every channel counts nanoseconds from its own creation): start_ns[cells]
 * in the clock of the t_ns / now_ns arguments; channel c then sees time t - start_ns[c] (subscription times, fan-out windows; ring
 * arrival times are channel times already).  NULL = one shared origin (the default). */
chd_status chd_set_channel_start_times(chd_engine* e, const int64_t* start_ns);

/* One fan-out decision = one fanOutDataUpdate call of the reference (data.go:221,263). */
#define CHD_DUE_VOID 0xFFFFFFFFu
typedef struct chd_due {
    uint32_t sub;          /* subscriber slot */
    uint32_t channel_id;   /* spatial channel */
    uint32_t kind;         /* 0 = FULL channel data (first fan-out, data.go:218-224), 1 = accumulated UPDATE,
                              CHD_DUE_VOID = not a decision (only in a list that overflowed, see CHD_OVF_DUE) */
    uint32_t n_selected;   /* UPDATE: ring entries merged (data.go:246-256) */
    uint32_t first_sel, last_sel; /* ring positions (0-based within the cell's ring) of the first/last merged entry */
    uint64_t sel_hash;     /* sum of merged entries' messageIndex mod 2^64 (lets the host verify its own selection) */
    uint64_t last_message_index; /* foc.lastMessageIndex after the step */
    int64_t  window_hi;    /* nextFanOutTime of the step: entries with lastUpdateTime <= arrival <= window_hi */
} chd_due;

/* ---- Channel.tickData for every spatial channel in one launch (data.go:175-291; replaces the per-channel
 * goroutine loop channel.go:358-387).  Per (subscriber, cell) pair: while t >= lastFanOutTime + interval
 * { first time: FULL, last = t; else select ring entries in [max(last,prev picked), last+interval] skipping
 * own updates, last += interval }.  All cells share one time origin (documented deviation: the reference
 * gives each channel its own startTime, channel.go:178).  Asynchronous. */
chd_status chd_fanout_tick(chd_engine* e, int64_t t_ns);

/* Counters of the work queued since the last summary; read back with ONE small device->host copy. */
typedef struct chd_tick_summary {
    uint64_t n_pairs;          /* live (subscriber, cell) subscriptions */
    uint64_t n_visible;        /* entries of the expanded visible list */
    uint32_t n_entities_in_world;
    uint32_t n_query_errors;
    uint32_t n_sub_new, n_unsub, n_kept;
    uint32_t n_due;
    uint32_t n_handover;
    uint32_t overflow;         /* bitmask of CHD_OVF_* (see below for what each one leaves behind) */
    uint64_t required_pairs, required_window_cells, required_visible;
    uint32_t required_due;
    uint32_t reserved;
} chd_tick_summary;
/* Capacities are fixed at chd_create, so an overflow cannot be retried with the same engine; what matters is that it never
 * corrupts state:
 *   CHD_OVF_PAIRS   the interest update was NOT applied: every subscriber keeps its previous subscriptions and fan-out state,
 *                   the diff lists are empty; required_pairs = the total the update would have needed
 *   CHD_OVF_WINDOW  the queries whose cell windows did not fit got CHD_Q_ERR_CAPACITY and, like any failed query, left their
 *                   subscribers untouched; the rest of the batch was applied, including every query with an empty window (spots
 *                   only, or shapes that miss the grid), which needs no scratch; required_window_cells = scratch needed
 *                   (either of these two on a tick whose batch came from chd_follow_queries(CHD_FOLLOW_MOVED): the followers'
 *                   stored centres advanced when the batch was generated, not when it was applied, so re-issue the tick's queries
 *                   with chd_follow_queries(CHD_FOLLOW_ALL); after chd_follow_queries_with(CHD_FOLLOW_MOVED, q), re-issue
 *                   chd_follow_queries_with(CHD_FOLLOW_ALL) with the same host part)
 *   CHD_OVF_VISIBLE the expanded visible list was not written (offsets are valid); required_visible = entries needed
 *   CHD_OVF_DUE     the pairs whose decisions did not fit were left untouched (still due: they catch up at the next
 *                   chd_fanout_tick); the list holds the decisions that did fit plus CHD_DUE_VOID holes; required_due
 *   CHD_OVF_BORDER  multi-GPU border / halo capacity exceeded: this tick's halo is incomplete */
enum { CHD_OVF_PAIRS = 1, CHD_OVF_WINDOW = 2, CHD_OVF_VISIBLE = 4, CHD_OVF_DUE = 8, CHD_OVF_BORDER = 16,
       CHD_OVF_RING = 32, /* a device-owned ring slab was full of live entries: its oldest entry was dropped */
       CHD_OVF_DELTA = 64, /* the visible-set delta did not fit chd_reserve_visible_delta's capacity: see chd_visible_delta */
       CHD_OVF_DELTA_IDS = 128 /* id-mode delta: an id >= id_space, or one id twice among one state's in-world entities; handled
                                  like CHD_OVF_DELTA (no lists, snapshot kept): see chd_reserve_visible_delta_ids */ };
/* bit 31: a device-side wait timed out (results invalid, please report).  A macro, not an enumerator: ISO C enumerators
 * must fit an int. */
#define CHD_OVF_INTERNAL 0x80000000u

/* Synchronises the stream and returns the counters.  CHD_ERR_CAPACITY if any overflow bit is set. */
chd_status chd_summary(chd_engine* e, chd_tick_summary* out);

/* ---- Channel.Tick for all spatial channels (channel.go:358-387), batched: build (if entities changed),
 * update_interest(q) (if q != NULL), emit_visible (flags & CHD_TICK_EMIT) and fanout_tick(t_ns) (flags & CHD_TICK_FANOUT),
 * with the results of those four calls in that order, then the summary.  No intermediate host sync.  Two streams: when
 * there is something to overlap, the interest update and the fan-out pass run on the engine's second stream next to build
 * + emit on the engine stream (the emit preparation waits only for the new pairs and the cell counts), and the engine
 * stream waits for the second one before the summary; otherwise the stages run one after the other on the engine stream. */
enum {
    CHD_TICK_BUILD = 1, CHD_TICK_EMIT = 2, CHD_TICK_FANOUT = 4, CHD_TICK_ALL = 7,
    /* The host will read this tick's results back (chd_fetch_results): start the expanded-list kernel only after the
     * fan-out pass (it would otherwise starve it of SM slots), so that every host-facing result is final, and is copied
     * to the host, while that kernel is still running.  Costs ~0.06 ms of device time per tick; results are identical. */
    CHD_TICK_EARLY_RESULTS = 8,
    /* Run chd_visible_delta after the build and the interest update (with or without CHD_TICK_EMIT).  In a two-stream tick it
     * runs on a third stream next to the expanded-list kernel and the fan-out pass; the engine stream waits for it. */
    CHD_TICK_VISIBLE_DELTA = 16,
    /* The tick's query batch is the one chd_follow_queries generated (pass q == NULL): the interest update consumes it as it
     * consumes a batch given in q.  CHD_ERR_STATE if no generated batch is waiting, CHD_ERR_INVALID together with q != NULL. */
    CHD_TICK_FOLLOW = 32
};
/* Optional early start: the interest update (and the fan-out pass when with_fanout != 0) do not depend on the entity
 * positions, so a host can start them as soon as the tick's queries and rings are known — on the engine's second
 * stream — and then upload / exchange positions; the following chd_tick(e, NULL, t_ns, flags, ..) runs build + emit
 * and joins.  Used by the multi-GPU driver to overlap the border exchange with the interest stage.
 * q == NULL (here and in chd_update_interest) = the batch uploaded by chd_prefetch_queries and handed over by
 * chd_adopt_prefetched, or the batch generated by chd_follow_queries; CHD_ERR_STATE if there is none. */
chd_status chd_begin_interest(chd_engine* e, const chd_query_batch* q, int64_t t_ns, int with_fanout);
/* Completion: after chd_tick returns, work the caller enqueues on the engine stream is ordered after every result of the tick
 * except the expanded list (vis_entity): in a two-stream tick the expanded-list kernel keeps running on a low-priority stream of
 * its own, next to the following tick's build, interest update and emit preparation.  The expanded list is final once any of
 * these has been called: chd_summary (also through out != NULL), chd_sync, any chd_get_*, chd_device_view, chd_fetch_results
 * with vis_entity != NULL, chd_build, chd_emit_visible, chd_update_interest, chd_fanout_tick, the payload, broadcast and
 * window-class calls, chd_tick_sharded, chd_destroy — or once the next chd_tick has returned.  The tick-path inputs
 * (chd_set_entities*, chd_set_rings, chd_prefetch_*, chd_adopt_prefetched, chd_begin_interest, chd_follow_queries*, the entity
 * events), chd_tick itself and chd_fetch_results_async* / chd_fetch_wait* do not wait for it. */
chd_status chd_tick(chd_engine* e, const chd_query_batch* q, int64_t t_ns, uint32_t flags, chd_tick_summary* out);

/* ---- results.  Each copies to caller memory (host or device) on the engine stream and synchronises.
 * Pass NULL for arrays you do not need.  Counts come from chd_summary. */
/* cell CSR: cell_start[cells+1], sorted_entity[n_entities_in_world] */
chd_status chd_get_cells(chd_engine* e, uint32_t* cell_start, uint32_t* sorted_entity);
/* subscriptions CSR by subscriber slot: pair_off[n_subscribers+1]; per pair channel id, dist, interval ms,
 * flags (bit0 hadFirstFanOut, bit1 subscribed by the last update_interest, bit2 skipSelf), lastFanOutTime */
chd_status chd_get_pairs(chd_engine* e, uint32_t* pair_off, uint32_t* channel_id, uint32_t* dist, uint32_t* interval_ms,
                         uint8_t* flags, int64_t* last_fanout_ns, uint64_t* last_message_index);
/* status per query of the last chd_update_interest batch */
chd_status chd_get_query_status(chd_engine* e, uint32_t* status, uint32_t n);
/* interest diff of the last update: (subscriber slot, channel id) lists.  They are SETS: the order is unspecified
 * (the reference issues these messages in Go map order); sort on the host if a canonical order is needed. */
chd_status chd_get_diff(chd_engine* e, uint32_t* new_sub, uint32_t* new_channel, uint32_t* unsub_sub, uint32_t* unsub_channel);
/* visible lists: vis_off[n_subscribers+1] (u64), vis_entity[n_visible] */
chd_status chd_get_visible(chd_engine* e, uint64_t* vis_off, uint32_t* vis_entity);
/* one subscriber's visible list: copies min(count, cap) entries, *count = its full length */
chd_status chd_get_visible_slot(chd_engine* e, uint32_t slot, uint32_t* out, uint64_t cap, uint64_t* count);
/* fan-out decisions of the last chd_fanout_tick.  A SET: the decisions of one (subscriber, channel) pair are contiguous
 * and in step order, the order across pairs is unspecified (the reference sends from independent channel goroutines). */
chd_status chd_get_due(chd_engine* e, chd_due* out, uint32_t cap);
/* handover candidates of the last build: entity, src channel id, dst channel id (0 = left/entered the world) */
chd_status chd_get_handover(chd_engine* e, uint32_t* entity, uint32_t* src_channel, uint32_t* dst_channel, uint32_t cap);

/* ---- visible-set deltas: which entities each subscriber slot should spawn / despawn, without reading the expanded lists back.
 * visible(s) is as for chd_emit_visible: the entities whose current cell is one of slot s's subscribed cells.  For every slot s
 *     entered(s) = visible_now(s) \ visible_snap(s)        left(s) = visible_snap(s) \ visible_now(s)
 * where "snap" is the engine state at the last delta that succeeded (before the first one every set is empty, so the first
 * delta enters the full visible lists).  A delta is measured against that snapshot, not against the previous tick: ticks run
 * without CHD_TICK_VISIBLE_DELTA, standalone chd_build / chd_update_interest calls and the subscriber lifecycle calls all fold
 * into the next delta.  So a removed slot (chd_remove_subscribers, chd_set_subscribers) leaves everything it saw, an added slot
 * enters what its first query makes visible, and a failed query (CHD_Q_ERR_*) changes nothing for its slot.
 * "now" is the state of the last chd_build and the current subscriptions; CHD_ERR_STATE if chd_assign_cells ran after that build.
 * Entity identity depends on the mode, which the first reserve call picks (index mode: chd_reserve_visible_delta, id mode:
 * chd_reserve_visible_delta_ids, below).  In index mode it is the entity index.  An index at or above the entity count of a state, or outside the world in it (NaN-parked
 * slots included), is absent from that state: appended spawns, a shrunk array and parked slots come out as enter / leave.  An
 * index reused for a different entity between two deltas is invisible to the engine: the host despawns / spawns it itself.
 * Order: entered(s) by (current cell asc, entity asc), left(s) by (snapshot cell asc, entity asc): the order of the visible
 * lists, so results are deterministic.
 *   chd_reserve_visible_delta  allocates the snapshot (about 8 bytes per entity of capacity) on the first call, which enables the
 *                              feature, and grows both output lists to cap_entries entries each.  Synchronous, not on the tick path;
 *                              the last delta's lists are discarded (they read as empty until the next delta).
 *   chd_visible_delta          computes the delta and advances the snapshot.  Stream-ordered, no host synchronisation.  If a list
 *                              needs more than the reserved capacity, CHD_OVF_DELTA is raised, nothing is written and the snapshot
 *                              is NOT advanced: after chd_reserve_visible_delta with the reported counts, the next delta covers
 *                              everything since the last successful one.
 *   chd_get_visible_delta      copies the last delta: enter_off / leave_off [*n_slots + 1] (u64 CSR by slot), the entities
 *                              [cap] each; n_entered / n_left = list lengths (also after an overflow: the required sizes).
 *                              *n_slots = max(slots now, slots at any earlier delta): slots dropped by chd_set_subscribers still
 *                              report what they left.  Synchronous; any pointer may be NULL; CHD_ERR_CAPACITY if a requested list
 *                              does not fit cap or the last delta overflowed.
 * Index mode is single-GPU only: CHD_ERR_STATE on an engine that has used chd_set_slab, chd_set_entity_ids or chd_comm_init (halo
 * entity indices are not stable from tick to tick there).
 *
 * Id mode: entity identity is the GLOBAL id (chd_set_entity_ids for own entities, the halo records of chd_import_halo /
 * chd_tick_sharded for the rest), not the entity index.  Works on single engines with ids, on slabs driven through the building
 * blocks and in chd_tick_sharded, and survives halo reordering, re-homing (own on one rank, halo on another, then own there) and a
 * host that permutes its entity array between deltas.  The lists name global ids; inside a cell they follow the cell CSR (own
 * entities in array order, then halo entities in import order), so, as for the multi-GPU visible lists, read each cell's part as a set.
 *   chd_reserve_visible_delta_ids  as chd_reserve_visible_delta, and picks id mode over the ids [0, id_space) (the snapshot takes
 *                                  8 bytes per id of id_space).  CHD_ERR_STATE after index mode was picked; later calls of either
 *                                  reserve function on an id-mode engine only grow the lists (a different id_space: CHD_ERR_INVALID).
 *                                  In entity-table mode it is the delta mode of an engine made a slab (chd_set_slab / chd_comm_init,
 *                                  a one-slab world included) before chd_entity_table_init: the table ids are the global ids, so
 *                                  every table id must be below id_space.  On a table engine that is not a slab: CHD_ERR_STATE (its
 *                                  index-mode deltas already name ids).
 * An id-mode delta needs ids for the own entities (chd_set_entity_ids or entity-table mode; CHD_ERR_STATE otherwise) and,
 * standalone, a chd_build after the last change of positions, ids, table or halo.  If an in-world entity of the current state has an id >= id_space, or two in-world entities share an id
 * (the host routed one entity to two places), CHD_OVF_DELTA_IDS is raised: no lists are written and the snapshot is not advanced,
 * so the next clean delta covers everything (chd_get_visible_delta then returns CHD_ERR_INVALID for the lists).  Entities outside
 * the world are absent and never count as duplicates.
 * Subscriber migration (chd_migrate_out / chd_migrate_in): the source rank's next delta reports the emigrant leaving everything its
 * snapshot held, the destination's reports the immigrant entering everything it sees; the host nets the two (enter = enter_B \
 * leave_A, leave = leave_A \ enter_B), exact when A's leave list is paired with B's first successful delta for that connection. */
chd_status chd_reserve_visible_delta(chd_engine* e, uint64_t cap_entries);
chd_status chd_reserve_visible_delta_ids(chd_engine* e, uint64_t cap_entries, uint32_t id_space);
chd_status chd_visible_delta(chd_engine* e);
chd_status chd_get_visible_delta(chd_engine* e, uint64_t* enter_off, uint32_t* enter_entity, uint64_t* leave_off, uint32_t* leave_entity,
                                 uint64_t cap, uint64_t* n_entered, uint64_t* n_left, uint32_t* n_slots);

/* ---- entity-table mode: entities as events keyed by id, as channeld delivers them (SpawnObjectMessage / DestroyObjectMessage,
 * pkg/unreal/message.go:20-203; a move is an ENTITY-channel update whose Merge hook calls Notify for that entity alone,
 * spatial.go:612-626).  The engine keeps the id -> slot map and assigns position slots itself; the host never sees a slot.
 *   chd_entity_table_init  switches a FRESH engine into table mode (CHD_ERR_STATE after any chd_set_entities* / chd_prefetch_entities*
 *                          / chd_assign_cells / chd_build, or after chd_set_entity_ids / chd_export_border /
 *                          chd_reserve_visible_delta_ids).  chd_set_slab / chd_comm_init may come first: that makes it a table
 *                          engine on slabs (below).  Allocates the device id table (2^k >= 2 x max_entities words) and the slot
 *                          -> id array, and parks every position slot (NaN: outside the world).  From then on these return
 *                          CHD_ERR_STATE: the calls that bypass the table (chd_set_entities*, chd_prefetch_entities*,
 *                          chd_entity_buffers, chd_set_entity_count, chd_set_entity_ids: the table ids ARE the global ids), and
 *                          chd_set_slab / chd_comm_init (the slab is fixed once the table exists).  chd_export_border,
 *                          chd_import_halo and chd_tick_sharded work on a table engine made a slab first, and return
 *                          CHD_ERR_STATE on one that was not: such an engine is single-GPU.
 *   chd_spawn_entities     AddEntity for each (id[i], x[i], z[i]); _f32: FVector positions, widened exactly as chd_set_entities_f32
 *                          widens them.  out_status[i] (may be NULL) is one CHD_EV_* per event, written before the call returns.
 *   chd_despawn_entities   RemoveEntity for each id[i]; out_status as for spawns.
 *   chd_move_entities      new positions of live ids (_f32: FVector positions).  If one call moves an id several times the LAST one
 *                          in array order wins (the reference applies updates in arrival order).  A move of an id that is not live
 *                          (reserved ids included) is ignored and counted.  Ids are resolved on the device.
 *   chd_get_entity_stats   synchronous counters (below).
 * Events are stream-ordered and apply in call order; pointer rules are those of chd_set_entities (host inputs are copied, device
 * inputs of a move are read in place; the ids and positions of a spawn / despawn are read on the host, a device array is copied back
 * first).  Statuses:
 *   reserved ids  0 and 0xFFFFFFFF are rejected (CHD_EV_RESERVED_ID; a NetGUID of 0 is invalid in the reference, message.go:40-43);
 *   duplicate     a spawn of a live id, or an id repeated in one spawn / despawn call (the first occurrence is applied);
 *   unknown id    a despawn of an id that is not live;
 *   table full    no slot is free (see the quarantine below).
 * A rejected event changes nothing.  A spawn outside the world is live but in no cell (the reference logs it and does not add it);
 * a later move into the world is reported as a handover from 0.
 * Results in table mode name IDS: the cell CSR's sorted_entity (chd_get_cells, chd_fetch_results*, CHD_VIEW_SORTED_ENTITY), the
 * visible lists, the handover list (chd_get_handover, the fetch paths, summary.n_handover) and the visible-set deltas.  Inside a
 * cell, entries are in slot order; slots are assigned deterministically (a released slot first in first out, then the next fresh
 * one), so the same event sequence gives identical arrays, with or without CUDA graphs.  The handover list holds the moved entities
 * whose cell changed since the previous build, including dst = 0 for leaving the world; entities spawned or despawned since then are
 * not in it (those are AddEntity / RemoveEntity, not Notify); after a standalone chd_assign_cells it names ids once the following
 * chd_build has run.  CHD_VIEW_ENTITY_ID gives the id of each slot (0 = empty) for
 * consumers that stay on the device.
 * Visible-set deltas work in table mode.  In index mode (chd_reserve_visible_delta, single-GPU) a despawned id that is spawned
 * again is a new instance, in `leave` (the old one) and in `enter` (the new one).  In id mode (chd_reserve_visible_delta_ids)
 * identity is the id: a despawn followed by a spawn of the same id between two deltas is NOT reported where a slot sees the id in
 * both states, and no slot is quarantined.  Index-mode slot quarantine keeps index mode exact: without chd_reserve_visible_delta a despawned slot may be reused by the
 * next spawn call; with it, only after a delta that ran after the despawn has SUCCEEDED, as observed by the library in a summary it
 * read (chd_summary, chd_tick with `out`, chd_fetch_results, chd_fetch_wait); after CHD_OVF_DELTA the slot stays quarantined.
 * Until a slot is released spawns take fresh ones, and when none is left the status is CHD_EV_TABLE_FULL.  A standalone
 * chd_visible_delta needs a chd_build after the last event (CHD_ERR_STATE otherwise; chd_tick builds first).
 * Table mode on slabs (chd_set_slab or chd_comm_init, then chd_entity_table_init): each rank's table holds the entities it OWNS;
 * every id is live on at most one rank.  Per tick: events -> chd_export_border (border records carry table ids) -> exchange ->
 * chd_import_halo -> chd_build / chd_tick, or events -> chd_tick_sharded; the events are stream-ordered before the tick and the
 * tick adds no host synchronisation.  Results name ids, own and halo alike.  The handover list reports each cell change once, by
 * the rank that owned the entity when it happened (the destination may be a cell of another slab); handover detection stays on
 * when ownership changes, because slots handed off (chd_handoff_entities) or adopted (a spawn) are flagged like despawns and
 * spawns: neither rank reports the hand-off itself, and a cell change of an adopted entity before its new owner's next cell
 * assignment is not reported either (it counts as the spawn's).  Id-mode deltas are the only delta mode on slabs; an id that goes
 * from halo to own (or back) while a slot sees it is in neither list. */
enum { CHD_EV_OK = 0, CHD_EV_DUPLICATE = 1, CHD_EV_UNKNOWN_ID = 2, CHD_EV_RESERVED_ID = 3, CHD_EV_TABLE_FULL = 4 };
typedef struct chd_entity_stats {
    uint32_t live;              /* ids spawned and not despawned */
    uint32_t high_water;        /* slots ever used (the entity count every build covers) */
    uint32_t quarantined;       /* despawned slots waiting for a successful visible delta */
    uint32_t free_slots;        /* slots a spawn could take now: released ones + max_entities - high_water */
    uint64_t moves_applied;     /* since chd_entity_table_init */
    uint64_t moves_unknown;     /* moves of ids that were not live */
    uint64_t moves_superseded;  /* moves overridden by a later move of the same id in the same call */
    uint64_t rebuilds;          /* device id-table rebuilds (live entries + tombstones passed 3/4 of the table) */
} chd_entity_stats;
chd_status chd_entity_table_init(chd_engine* e);
chd_status chd_spawn_entities(chd_engine* e, const uint32_t* id, const double* x, const double* z, uint32_t n, uint8_t* out_status);
chd_status chd_spawn_entities_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, uint32_t n, uint8_t* out_status);
chd_status chd_despawn_entities(chd_engine* e, const uint32_t* id, uint32_t n, uint8_t* out_status);
chd_status chd_move_entities(chd_engine* e, const uint32_t* id, const double* x, const double* z, uint32_t n);
chd_status chd_move_entities_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, uint32_t n);
chd_status chd_get_entity_stats(chd_engine* e, chd_entity_stats* out);

/* ---- followers: subscriber slots whose area of interest is centred on an entity ("a player stands on its pawn").  The engine
 * holds the positions already (after the tick's entity events or position upload), so it can build the tick's query batch itself:
 * the host binds slot -> (entity, AOI shape) once and then asks for the batch each tick, instead of mirroring every followed
 * entity's position and packing and uploading 28-33 bytes per subscriber per tick.
 *   chd_follow_bind     binds (or re-binds: that is how a shape or direction changes) slot[i] to entity[i] with the shape given by
 *                       kind[i], a mask out of CHD_AOI_SPHERE | CHD_AOI_BOX | CHD_AOI_CONE; every kind of one follower is centred
 *                       on the entity.  CHD_AOI_SPOTS has absolute positions and is refused.  entity[i] is the entity index; in
 *                       entity-table mode it is the table id (with chd_set_entity_ids, ids without a table, it stays the index).
 *                       A slot named twice in one call: the last one wins.  Arrays are HOST memory, copied before the call returns.
 *                       CHD_ERR_INVALID (nothing is bound): a slot that was never added (>= the slot count), a kind of 0 or with
 *                       other bits, a kind whose shape arrays are NULL; CHD_ERR_CAPACITY: more followers than
 *                       chd_limits.max_queries.  The per-slot state is allocated by the first call.
 *   chd_follow_unbind   the slots follow nothing from now on; their subscriptions stay as they are.  chd_remove_subscribers
 *                       unbinds the removed slots, chd_set_subscribers unbinds every slot.
 *   chd_follow_queries  generates the batch on the engine stream, ordered after every entity event / position upload or adoption
 *                       enqueued before it; asynchronous, no host synchronisation.  The batch is the one a host would have packed:
 *                       one query per selected follower, sub = its slot, centre = the f64 position the build reads for its entity
 *                       (after f32 widening, after the last-wins election of moves), shape from the binding, selected followers
 *                       in ascending slot order.  CHD_FOLLOW_ALL selects every follower whose entity exists.  CHD_FOLLOW_MOVED
 *                       selects a follower whose entity exists and whose binding is new or changed since the last batch that
 *                       selected it, or whose entity's position differs BITWISE from the centre of the last query generated for
 *                       it; skipping the others is sound, an identical query gives identical subscriptions (kept pairs keep their
 *                       fan-out state and interval, subscription.go:44-57).  A follower whose entity does not exist (index >= the
 *                       entity count; id not live in the table — a slot reused by another id is not followed) gets no query and
 *                       keeps its subscriptions, like a connection that sent no update; when the id is spawned again the follower
 *                       resumes and counts as moved.  On a slab (entity-table mode) the id resolves through the rank's own table,
 *                       which holds its own entities only, so "the entity exists" means "this rank owns it": a follower whose id is
 *                       a halo entity, or was handed off (chd_handoff_entities), gets CHD_FOLLOW_NO_ENTITY, keeps its
 *                       subscriptions, and counts as moved when the id is own again.  Also on a slab, a selected follower whose
 *                       query would reach columns the slab does not serve gets no query and CHD_FOLLOW_OUTSIDE_SLAB: the served
 *                       columns are [col_lo - halo, col_hi + halo); the query's span is the union over its kinds of the columns
 *                       floor((cx - reach - off_x) / w) .. floor((cx + reach - off_x) / w) (reach = sph_r, box_ex, cone_r), clipped
 *                       to [0, cols) because samples outside the world are skipped.  The check is conservative (a bounding box,
 *                       not the samples).  Such a follower keeps its subscriptions and its last centre, and counts as moved.  An
 *                       engine that is not a slab never makes this check.  An entity outside the world gives CHD_Q_ERR_OUT_OF_WORLD from the query
 *                       path as for any batch.  The batch has one entry per FOLLOWER (B): entries behind the selected ones are
 *                       skip entries (sub = 0xFFFFFFFF, kind = 0, status CHD_Q_OK), so the batch length the interest stage and
 *                       chd_get_query_status / the status list of chd_fetch_results* see is B, and entry i below the selected
 *                       count is the i-th selected follower in slot order.  No followers: an empty batch (which still applies
 *                       pending lifecycle changes).
 *                       The batch is handed over like an adopted prefetched batch: the next chd_begin_interest /
 *                       chd_update_interest with q == NULL, or chd_tick with CHD_TICK_FOLLOW, consumes it.  One batch per interest
 *                       update: CHD_ERR_STATE while an adopted prefetched batch or an earlier generated one is unconsumed, and
 *                       while a chd_begin_interest is pending; chd_adopt_prefetched of a query batch is refused while a generated
 *                       one is unconsumed.  Queries of subscribers that follow nothing join the batch through
 *                       chd_follow_queries_with.
 *   chd_follow_queries_with
 *                       chd_follow_queries(mode) plus a HOST PART: the explicit queries of the tick (spectators, free cameras,
 *                       SpotsAOI, cones that do not look along the pawn), merged with the generated ones into ONE batch on the
 *                       engine stream, so one interest update, one diff, one status list and one read-back cover the whole tick.
 *                       The host part is q, a batch exactly as chd_update_interest takes it (host or device arrays; device arrays
 *                       are read in place; sub must not be NULL), or, with q == NULL, the batch handed over by
 *                       chd_adopt_prefetched, which this call consumes.  The merged batch owns copies of everything it reads, so
 *                       the adopted staging set is free for the next chd_prefetch_queries once the merge has run.  Layout, with
 *                       n_h host entries, B followers, H = 0 if n_h == 0 else max(256, the next power of two >= n_h):
 *                         [0, n_h)               the host part, in the host's order
 *                         [n_h, H)               skip entries (sub = 0xFFFFFFFF, kind = 0, status CHD_Q_OK, no spots)
 *                         [H, H + n_selected)    the selected followers, in ascending slot order
 *                         [H + n_selected, H+B)  skip entries
 *                       The batch length, and the length of its status list, is H + B (size classes keep the length, and so the
 *                       stages' CUDA graphs, constant while the explicit count varies).  With n_h == 0 the call is
 *                       chd_follow_queries(mode), bit for bit.  A host entry behaves as it does in a batch of its own (statuses,
 *                       removed or unknown slots, spots, at most one entry per slot); an entry whose kind names arrays the host
 *                       part did not supply gets CHD_Q_ERR_MISSING_ARRAY even though the followers supply them.  A follower slot
 *                       with a host entry is OVERRIDDEN for this tick: its explicit query wins, it gets no generated query
 *                       (chd_get_follow reports CHD_FOLLOW_OVERRIDDEN), its stored centre stays, and it counts as moved, so the
 *                       next CHD_FOLLOW_MOVED generation selects it again and its subscriptions return to the follow shape (unbind
 *                       the slot to keep the explicit query).  Consumed like chd_follow_queries' batch.  Refused, changing nothing
 *                       (an adopted batch stays adopted): CHD_ERR_CAPACITY if H + B > max_queries; CHD_ERR_STATE on an index-mode or id-mode slab,
 *                       while a generated batch is unconsumed or a chd_begin_interest is pending, with q == NULL and no adopted
 *                       query batch, and with q != NULL while an adopted one is unconsumed; CHD_ERR_INVALID for a bad mode or a
 *                       host part with sub == NULL.
 *   chd_get_follow      after the interest update that consumed the batch (and before the next one): per follower, in ascending
 *                       slot order, its slot, entity, the centre of the last query generated for it, and status = the CHD_Q_*
 *                       status of its query (its entry in a merged batch is H + its rank), or CHD_FOLLOW_NOT_SELECTED /
 *                       CHD_FOLLOW_NO_ENTITY / CHD_FOLLOW_OVERRIDDEN / CHD_FOLLOW_OUTSIDE_SLAB.  *count = followers (copies
 *                       min(count, cap)), *n_selected = queries in the last generated batch; this call is where the selected count
 *                       is reported (chd_tick_summary is unchanged).  Synchronous; any pointer may be NULL.
 * Followers on a slab need entity-table mode (the slab first, then chd_entity_table_init): a follower lives on the rank that owns
 * its entity, whose exact position is local there (border records carry no positions).  CHD_ERR_STATE on an index-mode or id-mode
 * slab, and chd_set_slab / chd_comm_init are refused once a slot follows.  chd_tick_sharded(e, NULL, .., flags | CHD_TICK_FOLLOW)
 * consumes the generated batch as chd_tick does.  A follower moves with its entity: chd_migrate_out unbinds the emigrants, and the
 * destination binds them again with chd_follow_bind after chd_migrate_in (the binding does not travel in the migration blob).
 * Halo: halo_cols >= ceil(max reach / w) + the columns an entity can cross in one tick keeps the tick on which an entity crosses
 * into a neighbour's slab exact (its old owner still generates the query); a smaller halo reports CHD_FOLLOW_OUTSIDE_SLAB there.
 * Not supported: centre offsets, cone directions taken from an entity's rotation, spots relative to an entity. */
typedef struct chd_follow_batch {          /* SoA, HOST arrays */
    uint32_t n;
    const uint32_t* slot;                  /* [n] subscriber slot */
    const uint32_t* entity;                /* [n] entity index, or table id in entity-table mode */
    const uint8_t*  kind;                  /* [n] CHD_AOI_SPHERE | BOX | CONE mask, NULL = all CHD_AOI_SPHERE */
    const double *sph_r, *box_ex, *box_ez, *cone_dx, *cone_dz, *cone_angle, *cone_r; /* [n] each; NULL if no binding uses the kind */
} chd_follow_batch;
enum { CHD_FOLLOW_ALL = 0, CHD_FOLLOW_MOVED = 1 };
enum { CHD_FOLLOW_NOT_SELECTED = 16, CHD_FOLLOW_NO_ENTITY = 17 }; /* beside CHD_Q_* in chd_get_follow's status */
enum { CHD_FOLLOW_OVERRIDDEN = 18 };  /* the slot's host entry in chd_follow_queries_with's batch replaced its generated query */
enum { CHD_FOLLOW_OUTSIDE_SLAB = 19 }; /* the generated query would reach columns the slab does not serve: no query this tick */
chd_status chd_follow_bind(chd_engine* e, const chd_follow_batch* b);
chd_status chd_follow_unbind(chd_engine* e, const uint32_t* slot, uint32_t n);
chd_status chd_follow_queries(chd_engine* e, uint32_t mode);
chd_status chd_follow_queries_with(chd_engine* e, uint32_t mode, const chd_query_batch* q);
chd_status chd_get_follow(chd_engine* e, uint32_t* slot, uint32_t* entity, uint32_t* status, double* cx, double* cz, uint32_t cap,
                          uint32_t* count, uint32_t* n_selected);

/* ---- all host-facing results of a tick in ONE call instead of one or two synchronisations per getter.  After a
 * two-stream tick (chd_tick with emit, or chd_begin_interest + chd_tick) the lists are copied in the order they become
 * final, on the engine's read-back streams, while the expanded-list kernel may still be running: first the pairs /
 * sub-unsub lists / query statuses / handover list / cell CSR (after the interest fill and the build), then the due list
 * and the visible offsets (after the fan-out pass, the emit preparation and, with CHD_TICK_VISIBLE_DELTA, the delta, whose
 * CHD_OVF_DELTA belongs to this summary; see CHD_TICK_EARLY_RESULTS); the call returns
 * when the tick has finished.  Otherwise: waits for the tick, reads the summary, enqueues every copy, waits once.
 * Exact sizes come from the device counters.  Any pointer may be NULL (skipped).  Capacities are in elements; CHD_ERR_CAPACITY if a requested list does not
 * fit (nothing is truncated silently).  This is what a channeld host calls once per tick. */
typedef struct chd_result_buffers {
    uint32_t *pair_off, *pair_channel, *pair_dist, *pair_interval_ms; /* pair_off[n_subscribers+1]; others [pair_cap] */
    uint64_t pair_cap;
    uint32_t *new_sub, *new_channel, *unsub_sub, *unsub_channel;      /* [diff_cap] each */
    uint64_t diff_cap;
    chd_due* due;                                                     /* [due_cap] */
    uint32_t due_cap;
    uint32_t *handover_entity, *handover_src, *handover_dst;          /* [handover_cap] */
    uint32_t handover_cap;
    uint32_t* query_status;                                           /* [status_cap] */
    uint32_t status_cap;
    uint64_t* vis_off;                                                /* [n_subscribers+1] */
    uint32_t* vis_entity;                                             /* [vis_cap] (the big one: usually NULL) */
    uint64_t vis_cap;
    uint32_t *cell_start, *sorted_entity;                             /* [cells+1], [entity_cap] */
    uint32_t entity_cap;
} chd_result_buffers;
chd_status chd_fetch_results(chd_engine* e, const chd_result_buffers* bufs, chd_tick_summary* summary);

/* ---- the same read-back WITHOUT blocking: copy kernels that know the exact lengths on the device first snapshot the lists into a
 * staging area in HBM (microseconds; the next tick's kernels are ordered after THIS, not after the PCIe transfer), then write the
 * snapshot into the caller's PINNED host buffers (chd_alloc_pinned) on a stream of their own; the call returns at once, so the host
 * can enqueue the NEXT tick before looking at this one.
 * pinned_header: CHD_FETCH_HEADER_BYTES of pinned memory the engine uses for the counters.  Up to two fetches may be outstanding
 * (use two sets of buffers); chd_fetch_wait blocks until the copies of the OLDEST outstanding chd_fetch_results_async are
 * complete and returns that tick's summary (CHD_ERR_CAPACITY if a list did not fit its
 * buffer: it was truncated to the capacity).  vis_entity is not supported here (the expanded list stays in HBM).
 * Loop of a pipelined host:  prefetch(k+1) ... adopt, chd_begin_interest, chd_tick(k) ; chd_fetch_results_async(k) ;
 * [enqueue tick k+1 the same way] ; chd_fetch_wait -> results of tick k while tick k+1 runs. */
#define CHD_FETCH_HEADER_BYTES 256
chd_status chd_fetch_results_async(chd_engine* e, const chd_result_buffers* bufs, void* pinned_header);
chd_status chd_fetch_wait(chd_engine* e, chd_tick_summary* summary);

/* ---- the visible-set delta read back with the tick's other results (the three calls above are these with delta == NULL).
 * Which delta: a fetch (sync or async) carries the most recent delta enqueued since the previous fetch on this engine, by
 * CHD_TICK_VISIBLE_DELTA (chd_tick, chd_tick_sharded) or by a standalone chd_visible_delta.  counts->deltas says how many were
 * enqueued: 0 = none (the counts are 0 and no delta buffer is written), 1 = these are its lists, > 1 = these are the last one's
 * lists and the earlier ones were never fetched (the host lost them).  With deltas >= 1 the offsets and lists equal what
 * chd_get_visible_delta returns right after that delta, in index, id and entity-table mode.
 * Overflow: after CHD_OVF_DELTA or CHD_OVF_DELTA_IDS the counts are the required sizes and no offsets or entries are copied; the
 * summary carries the bit and the call (sync) or chd_fetch_wait_delta (async) returns CHD_ERR_CAPACITY.
 * Caller capacity: slot_cap counts offsets (n_slots + 1 are needed for each CSR), entity_cap entries of each list.  If a requested
 * buffer is too small, the sync form copies no delta buffer and returns CHD_ERR_CAPACITY; the async form truncates to the capacity
 * and chd_fetch_wait_delta returns CHD_ERR_CAPACITY.
 * Any pointer may be NULL (delta == NULL: no delta read-back).  The async form needs pinned memory for every non-NULL buffer.
 * Delta buffers before any chd_reserve_visible_delta*: CHD_ERR_STATE.  chd_fetch_wait_delta may wait on any fetch (counts may be
 * NULL); a fetch issued without delta buffers reports deltas = 0.  The async counts ride in the pinned header.
 * Device memory: the async form snapshots the delta into the same HBM staging as the other lists, so each of its two staging sets
 * grows to up to 8 x entity_cap + 16 x slot_cap bytes more.  The snapshot starts when the delta is done, beside the expanded-list
 * kernel; only the next delta (and chd_reserve_visible_delta*) waits for it, the next tick's other stages do not. */
typedef struct chd_delta_buffers {
    uint64_t *enter_off, *leave_off;        /* [slot_cap] each: n_slots + 1 offsets */
    uint32_t *enter_entity, *leave_entity;  /* [entity_cap] each */
    uint64_t slot_cap, entity_cap;
} chd_delta_buffers;
typedef struct chd_delta_counts {
    uint64_t n_entered, n_left; /* list lengths; after CHD_OVF_DELTA(_IDS), the required sizes */
    uint32_t n_slots;           /* as chd_get_visible_delta's *n_slots */
    uint32_t deltas;            /* deltas enqueued since the previous fetch (see above) */
} chd_delta_counts;
chd_status chd_fetch_results_delta(chd_engine* e, const chd_result_buffers* bufs, const chd_delta_buffers* delta, chd_tick_summary* summary,
                                   chd_delta_counts* counts);
chd_status chd_fetch_results_async_delta(chd_engine* e, const chd_result_buffers* bufs, const chd_delta_buffers* delta, void* pinned_header);
chd_status chd_fetch_wait_delta(chd_engine* e, chd_tick_summary* summary, chd_delta_counts* counts);

/* Device-resident views (valid until the next call that rewrites them) for consumers that stay on the GPU. */
enum {
    CHD_VIEW_CELL_START = 0, CHD_VIEW_SORTED_ENTITY, CHD_VIEW_ENT_CELL, CHD_VIEW_PAIR_OFF, CHD_VIEW_PAIR_CHANNEL,
    CHD_VIEW_PAIR_DIST, CHD_VIEW_VIS_OFF, CHD_VIEW_VIS_ENTITY, CHD_VIEW_DUE,
    /* the visible-set delta (chd_visible_delta): u64 offsets [slots + 1] and u32 entities [capacity] of each list */
    CHD_VIEW_DELTA_ENTER_OFF, CHD_VIEW_DELTA_ENTER, CHD_VIEW_DELTA_LEAVE_OFF, CHD_VIEW_DELTA_LEAVE,
    /* entity-table mode: u32 id of each slot [high-water mark], 0 = empty */
    CHD_VIEW_ENTITY_ID
};
chd_status chd_device_view(chd_engine* e, int which, void** d_ptr, uint64_t* count);

/* ---- multi-GPU X-slab sharding (SURVEY.md §8e).  The engine owns grid columns [col_lo, col_hi) and serves
 * queries whose cells lie in [col_lo-halo, col_hi+halo).  After chd_build, chd_export_border writes the
 * (entity id, cell index) records of the entities in this rank's outermost `halo` columns on each side into a
 * caller-provided DEVICE buffer (2 x u32 per record; the unused tail is padded with 0xFFFFFFFF) for the all-gather;
 * chd_import_halo takes the gathered records of all ranks (records [skip_first, skip_first+skip_count) are this
 * rank's own and ignored), keeps those whose column lies in [col_lo-halo, col_hi+halo) and appends them as
 * position-less halo entities; the following chd_build sorts own + halo entities into the cell CSR.
 * Call order per tick: chd_set_entities -> chd_export_border (runs chd_assign_cells) -> all-gather ->
 * chd_import_halo -> chd_build.  Entity ids are global: set with chd_set_entity_ids, or the table ids in entity-table mode
 * (spawn / move / despawn events take the place of chd_set_entities there). */
chd_status chd_set_slab(chd_engine* e, uint32_t col_lo, uint32_t col_hi, uint32_t halo);
chd_status chd_set_entity_ids(chd_engine* e, const uint32_t* global_id, uint32_t n);
/* out_count may be NULL: then nothing synchronises with the host (an overflow of cap_records or of the entity capacity
 * surfaces as CHD_OVF_BORDER in the next chd_summary). */
chd_status chd_export_border(chd_engine* e, uint32_t* d_records, uint32_t cap_records, uint32_t* out_count);
chd_status chd_import_halo(chd_engine* e, const uint32_t* d_records, uint32_t n_records, uint32_t skip_first, uint32_t skip_count);

/* ---- the exchange behind the ABI: NCCL over NVLink / NVSwitch, one process per GPU.  libnccl.so.2 is loaded on first use
 * (a copy the process already holds is reused); a host needs no NCCL binding of its own.
 *   rank 0:      chd_comm_unique_id(id)            -> the host distributes the 128 bytes by any means (TCP, a file, MPI, ...)
 *   every rank:  chd_comm_init(e, id, rank, world, halo_cols, border_capacity, migrate_subscribers, migrate_pairs)   (collective;
 *                also sets this rank's slab: columns [floor(rank*cols/world), floor((rank+1)*cols/world)), halo_cols =
 *                ceil(max radius / grid_width); migrate_* = capacity of the per-tick subscriber migration blob, 0 = none)
 *   every tick:  chd_set_rings / chd_set_entities (this rank's entities, global ids via chd_set_entity_ids) ...
 *                chd_tick_sharded(e, q, t_ns, flags, summary) = chd_begin_interest + chd_export_border + ONE ncclAllGather of
 *                (entity id, cell) records (border_capacity records per rank, padded) + chd_import_halo + chd_tick: collective,
 *                stream-ordered, no host synchronisation unless summary != NULL.
 * border_capacity bounds the records ONE rank exports per tick (entities in its outermost halo_cols columns on each side
 * plus entities that left its slab); border_capacity * world must fit chd_limits.max_entities together with the own
 * entities.  Exceeding it raises CHD_OVF_BORDER. */
#define CHD_COMM_ID_BYTES 128
chd_status chd_comm_unique_id(void* out_id);
chd_status chd_comm_init(chd_engine* e, const void* unique_id, int rank, int world, uint32_t halo_cols, uint32_t border_capacity,
                         uint32_t migrate_subscribers, uint32_t migrate_pairs);
chd_status chd_comm_info(const chd_engine* e, int* rank, int* world, uint32_t* col_lo, uint32_t* col_hi, uint32_t* halo_cols, int* nccl_version);
chd_status chd_comm_destroy(chd_engine* e);
chd_status chd_tick_sharded(chd_engine* e, const chd_query_batch* q, int64_t t_ns, uint32_t flags, chd_tick_summary* out);
uint64_t chd_collective_count(const chd_engine* e); /* NCCL collectives issued so far */
/* How chd_tick_sharded moves the border records: 2 = PEER WINDOWS (default when every rank could map every other rank's receive
 * window with CUDA IPC at chd_comm_init: the export kernel's successor stores the live records straight into the peers' memory over
 * NVLink and publishes a 64-bit flag; the import's first kernel polls the local flags — no collective call on the tick path),
 * 1 = one ncclAllGather per tick (ranks without a P2P path, more than 16 ranks), 0 = no communicator.
 * chd_comm_use_collective(e, 1) selects the NCCL exchange even when peer windows are mapped (every rank must make the same choice,
 * between ticks); (e, 0) returns to the peer windows. */
int chd_comm_exchange_mode(const chd_engine* e);
chd_status chd_comm_use_collective(chd_engine* e, int on);

/* ---- re-homing.  ENTITIES: an entity that leaves its owner's slab is still exported by that owner and adopted, for this tick, by
 * every rank that needs it (visibility stays exact whatever the ownership); chd_get_rehome lists the own entities whose column
 * now belongs to another rank (global id, destination rank) so the host can re-route their position feed — the sender drops
 * them from its next chd_set_entities, the receiver includes them (the reference moves an entity between spatial channels the
 * same way, spatial.go:683-736).  In entity-table mode the host holds no positions: after the tick, chd_handoff_entities lists
 * those entities with their positions and removes them from the sender's table, and the receiver adopts them with
 * chd_spawn_entities before its next tick; moves and despawns of an id go to its current owner from then on.
 * SUBSCRIBERS live on the rank that owns their centre's column (the host routes each query there).  When that owner changes
 * from rank A to rank B the subscriber's subscriptions and fan-out state (lastFanOutTime, hadFirstFanOut, lastMessageIndex per
 * channel) travel INSIDE the tick's all-gather, so nothing is reset and nobody is re-sent FULL channel data:
 *   on A, before chd_tick_sharded:  chd_migrate_out(eA, slot[], n)          record i of A's blob = state of slot[i]; A's slots are
 *                                                                           freed by this tick's interest update (no unsub entries)
 *   on B, before chd_tick_sharded:  chd_migrate_in(eB, A, first_index, slot[], conn_id[], n)
 *                                   B's slot[i] becomes connection conn_id[i] with the state of record first_index + i of A's blob;
 *                                   its query in this tick's batch is diffed against that state.
 * Both ranks pass a query batch (an empty one will do) to the same chd_tick_sharded.  One chd_migrate_out per tick and rank;
 * any number of chd_migrate_in.  Capacities: chd_comm_init's migrate_* (overflow: CHD_OVF_BORDER, the cut-off subscribers arrive
 * without state).  slot / conn_id are HOST arrays. */
chd_status chd_migrate_out(chd_engine* e, const uint32_t* slot, uint32_t n);
chd_status chd_migrate_in(chd_engine* e, uint32_t src_rank, uint32_t first_index, const uint32_t* slot, const uint32_t* conn_id, uint32_t n);
/* own entities (of the last cell assignment) whose column lies outside this rank's slab: global id (entity-table mode: table id) +
 * the rank that owns the column now.  Synchronous and read-only.  *count = how many there are (copies min(count, cap)). */
chd_status chd_get_rehome(chd_engine* e, uint32_t* global_id, uint32_t* dst_rank, uint32_t cap, uint32_t* count);
/* Entity-table mode on slabs: hands the entities chd_get_rehome would list to their new owners.  Lists the own live in-world
 * entities of the last cell assignment whose column lies outside [col_lo, col_hi): id[i], dst_rank[i] (as chd_get_rehome computes
 * it) and the exact f64 position x[i], z[i]; and removes them from this rank's table (tombstone, slot -> id cleared, the slot
 * parked, flagged and released at once to the free-slot FIFO: the id lives on elsewhere, so no quarantine; `live` drops).  This
 * is not a despawn: the receiving rank adopts each entity with chd_spawn_entities(id, x, z), and the position arrives bit-exact.
 * Synchronous and transactional: *count = the number of entities eligible; if *count > cap, CHD_ERR_CAPACITY and nothing is
 * removed (a repeat call with a larger buffer lists the same set).  The output arrays may be host or device memory; they may be
 * NULL only with cap = 0.  CHD_ERR_STATE outside table mode, before any cell assignment, and after a spawn / move / despawn /
 * hand-off since the last assignment (the positions could be stale).  Call it once per tick, after the tick. */
chd_status chd_handoff_entities(chd_engine* e, uint32_t* id, uint32_t* dst_rank, double* x, double* z, uint32_t cap, uint32_t* count);

/* ---- window classes of the last fan-out pass (SURVEY.md §8f rank 1: payload assembly).  The reference merges the selected
 * update window afresh for every subscriber (data.go:248-252); decisions of one channel whose merged payload is
 * necessarily identical are grouped so the host merges / frames each distinct payload once:
 *   - all FULL decisions (kind 0) of a channel form one class (they all send ch.data.msg, data.go:219-224);
 *   - UPDATE decisions (kind 1) of a channel with the same lastFanOutTime at the start of the step, the same window_hi and
 *     no own update left out by SkipSelfUpdateFanOut form one class (the selection loop data.go:226-256 is then a
 *     function of the channel's buffer and these two times only);
 *   - an UPDATE decision whose subscriber had own updates inside the window is a class of its own.
 * out_class_of[i] = class of due record i (index into the list chd_get_due / chd_fetch_results return, same order),
 * out_class_rep[k] = lowest due index of class k (classes are numbered by it), out_class_count[k] = its size.
 * A CHD_DUE_VOID hole (a list that overflowed, CHD_OVF_DUE) has class CHD_DUE_VOID and is in no class: the classes, their
 * numbering, reps and counts cover the real decisions only.
 * Any output may be NULL.  CHD_ERR_CAPACITY if there are more than cap_classes classes.  Synchronous. */
chd_status chd_due_classes(chd_engine* e, uint32_t* out_class_of, uint32_t* out_class_rep, uint32_t* out_class_count,
                           uint32_t cap_classes, uint32_t* out_n_classes);

/* ---- the BYTE half of the fan-out (SURVEY.md §8f rank 1 and 4): per window class the wire bytes of its CHANNEL_DATA_UPDATE
 * message are assembled ONCE on the device (the reference re-merges and marshals three times per subscriber: data.go:246-256,
 * :295, connection.go:58, :671), then every connection's packets are laid out framed — 'C' 'H' size_hi size_lo compressionType
 * + marshalled Packet, optionally snappy-compressed (connection.go:626-714) — ready for conn.Write.
 *   chd_set_payload_bytes   per-tick input next to chd_set_rings: serialized updateMsg of every ring entry (CSR entry_off[n_entries+1]
 *                           in the ring order of chd_set_rings) and serialized full data message of every channel (full_off[cells+1]),
 *                           the Any type URL of the channel data type and the message type (MessageType_CHANNEL_DATA_UPDATE = 8).
 *   chd_assemble_payloads   after chd_fanout_tick / chd_tick: window classes (chd_due_classes) + for class k the bytes
 *                           blob[class_off[k] .. class_off[k+1]) = one Packet.messages entry (0x0A len MessagePack{channelId,
 *                           msgType, msgBody = ChannelDataUpdateMessage{data = Any{type_url, value}}}) where value = the
 *                           concatenation of the selected ring entries' bytes (= proto.Merge of them, by the protobuf encoding
 *                           rules) or the channel's full data for a FULL send.  Fields equal to 0 or empty are omitted as proto3
 *                           Marshal omits them, so the entry is byte for byte the protobuf serialization of that Packet.
 *                           Outputs may be NULL (results stay on the GPU).
 *   chd_frame_packets       per connection (subscriber slot s): bytes out[conn_off[s] .. conn_off[s] + conn_len[s]) = its packets
 *                           back to back, each 5-byte tag + body, messages in ascending due index; a packet holds as many of
 *                           the connection's messages as fit MaxPacketSize (0xffff), a message whose MessagePack is
 *                           >= MaxPacketSize - 5 bytes is dropped (connection.go:73-77; counted in *n_dropped); compression[s] = 1
 *                           -> snappy block format (decodes with any snappy decoder; the bytes differ from Go's encoder).
 *                           Deviation: a packet whose snappy encoding would exceed MaxPacketSize is sent uncompressed, with
 *                           compressionType 0 in its tag (readers decide per packet from the tag: connection.go:497-513,
 *                           client.go:208).  The reference writer refuses such a packet (connection.go:688-691) and its messages
 *                           are lost; Go's encoder rarely produces one, this engine's simpler encoder can on incompressible
 *                           bodies near 64 KB.  conn_off is spaced for the worst case; conn_frames[s] = packets written.
 * Valid for channel data types merged by the default reflection merge without ChannelDataMergeOptions (data.go:326-388);
 * types with a custom Merge stay on the host.  Synchronous; buffers of this stage grow on demand. */
chd_status chd_set_payload_bytes(chd_engine* e, const uint64_t* entry_off, uint32_t n_entries, const uint8_t* entry_bytes, const uint64_t* full_off,
                                 const uint8_t* full_bytes, const char* type_url, uint32_t msg_type);
chd_status chd_assemble_payloads(chd_engine* e, uint32_t* n_classes, uint64_t* class_off, uint32_t cap_classes, uint8_t* blob, uint64_t blob_cap,
                                 uint64_t* blob_len);
chd_status chd_frame_packets(chd_engine* e, const uint8_t* compression, uint64_t* conn_off, uint32_t* conn_len, uint32_t* conn_frames, uint8_t* out,
                             uint64_t out_cap, uint64_t* out_len, uint32_t* n_dropped);

/* ---- BroadcastType_ADJACENT_CHANNELS recipient sets, batched (message.go:188-239; SURVEY.md §8f rank 3).
 * For message m sent to spatial channel channel_id[m] with BroadcastType mask broadcast[m] (channeld.proto: ALL_BUT_SENDER 4,
 * ALL_BUT_OWNER 8, ALL_BUT_CLIENT 16, ALL_BUT_SERVER 32; the ADJACENT_CHANNELS bit itself is implied): the recipients are
 * the subscribers (slots of chd_set_subscribers, per the CURRENT spatial subscriptions = last chd_update_interest) of the
 * channel's 3x3 neighbours (spatial.go:358-381) and — unless ALL_BUT_OWNER — of the channel itself, each slot once
 * (the reference's adjacentConns map), minus the slot whose connection id equals sender_conn_id[m] when ALL_BUT_SENDER
 * is set, the clients / servers when ALL_BUT_CLIENT / ALL_BUT_SERVER are set (chd_set_subscriber_types), and the slot
 * whose connection id equals client_conn_id[m] (ServerForwardMessage.ClientConnId; 0 = none).
 * Output: CSR out_off[n + 1] / out_slot[] (a SET per message: the reference iterates a Go map), out_status[m] =
 * CHD_BC_OK or CHD_BC_ERR_NOT_A_CELL (channel id outside this grid: the reference cannot reach this, the channel must
 * exist; such a message gets no recipients).  Synchronous; CHD_ERR_CAPACITY if the lists need more than cap entries.
 * sender_conn_id / client_conn_id may be NULL (= all 0). */
typedef struct chd_broadcast_batch {
    uint32_t n;
    const uint32_t* channel_id;
    const uint32_t* broadcast;
    const uint32_t* sender_conn_id;
    const uint32_t* client_conn_id;
} chd_broadcast_batch;
enum { CHD_BC_OK = 0, CHD_BC_ERR_NOT_A_CELL = 1 };
enum { CHD_CONN_SERVER = 1, CHD_CONN_CLIENT = 2 }; /* channeldpb.ConnectionType */
/* ConnectionType per subscriber slot (NULL = unknown: the ALL_BUT_CLIENT / ALL_BUT_SERVER filters then remove nobody). */
chd_status chd_set_subscriber_types(chd_engine* e, const uint8_t* conn_type, uint32_t n);
chd_status chd_adjacent_broadcast(chd_engine* e, const chd_broadcast_batch* b, uint32_t* out_status, uint32_t* out_off,
                                  uint32_t* out_slot, uint64_t cap);

/* ---- control-plane helpers kept for interface completeness (pure integer/config math on the host; not part
 * of the data-parallel path): GetAdjacentChannels (spatial.go:358-381) and GetRegions (spatial.go:319-356). */
uint32_t chd_get_adjacent_channels(const chd_grid_cfg* cfg, uint32_t channel_id, uint32_t* out8);
chd_status chd_get_regions(const chd_grid_cfg* cfg, double* min_x, double* min_z, double* max_x, double* max_z,
                           uint32_t* channel_id, uint32_t* server_index);
/* dist -> FanOutIntervalMs (message_spatial.go:16-38); the same table the kernels use. */
uint32_t chd_damping_interval_ms(uint32_t dist, uint32_t default_ms);

/* ---- instrumentation.  chd_launch_count: kernels launched by this engine so far.  chd_profile_enable(1)
 * makes every stage record a CUDA-event pair on the engine stream (the last 1024 samples are kept);
 * chd_profile_get synchronises and returns the summed device time of a stage.  CHD_STAGE_EMIT_KERNEL brackets
 * exactly the emit_visible kernel (the dominant HBM term; bench.py's roofline uses it); chd_profile_enable(2) records that
 * pair only (two events per tick instead of about twenty: what bench.py leaves on inside its timed region). */
enum { CHD_STAGE_BUILD = 0, CHD_STAGE_INTEREST, CHD_STAGE_EMIT, CHD_STAGE_EMIT_KERNEL, CHD_STAGE_FANOUT, CHD_STAGE_TICK,
       CHD_STAGE_EXPORT, CHD_STAGE_EXCHANGE, CHD_STAGE_IMPORT, /* the three steps of chd_tick_sharded before the tick proper */
       CHD_STAGE_READBACK,                                     /* chd_fetch_results_async: the PCIe hop (snapshot -> pinned host) */
       CHD_STAGE_VISIBLE_DELTA,                                /* chd_visible_delta / CHD_TICK_VISIBLE_DELTA */
       CHD_STAGE_ENTITY_EVENTS,                                /* chd_spawn_entities* / chd_move_entities* / chd_despawn_entities */
       CHD_STAGE_FOLLOW,                                       /* chd_follow_queries */
       CHD_STAGE_COUNT };
uint64_t chd_launch_count(const chd_engine* e);
/* The launch-bound stages (build, interest update, emit preparation, fan-out) are replayed as CUDA graphs once
 * their shape (entity / query / subscriber counts) has been stable for two ticks.  chd_enable_graphs(e, 0) forces
 * direct launches; chd_graph_launch_count reports how many stage executions were graph replays. */
chd_status chd_enable_graphs(chd_engine* e, int on);
uint64_t chd_graph_launch_count(const chd_engine* e);
chd_status chd_profile_enable(chd_engine* e, int on);
chd_status chd_profile_get(chd_engine* e, int stage, double* total_ms, uint64_t* samples);
/* Timeline of the most recent chd_tick: start / stop of a stage in ms after the tick started (CHD_STAGE_TICK start). */
chd_status chd_profile_timeline(chd_engine* e, int stage, double* start_ms, double* stop_ms);

uint32_t chd_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif
