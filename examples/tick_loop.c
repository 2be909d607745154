/* tick_loop.c — the C ABI as a host sees it (plain C99; what the cgo shim in go/gpucontroller.go does, minus Go).
 * One engine, the pipelined tick loop of INTEGRATION.md §2: while tick k runs on the GPU the inputs of tick k+1 are
 * uploaded, and the results of tick k-1 are consumed (chd_fetch_results_async_delta / chd_fetch_wait_delta: the host never waits
 * for a tick before it has enqueued the next one), the visible-set delta (entities each subscriber spawns / despawns) among them.
 *
 *   gcc -std=c99 -Iinclude examples/tick_loop.c -Lchanneld_b200 -lchd_b200 -Wl,-rpath,$PWD/channeld_b200 -lm -o tick_loop
 *
 * tests/test_abi.py compiles and links this file on every run (it needs an H100 to actually execute).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "chd_gpu.h"

#define CHECK(call)                                                              \
    do {                                                                         \
        chd_status st_ = (call);                                                 \
        if (st_ != CHD_OK) {                                                     \
            fprintf(stderr, "%s -> %d: %s\n", #call, (int)st_, chd_last_error(e)); \
            return 1;                                                            \
        }                                                                        \
    } while (0)

/* two sets of page-locked staging buffers: the engine reads set (k+1)&1 while the host may already refill set k&1 */
typedef struct staging {
    double *x, *z;             /* entity positions */
    double *cx, *cz, *r;       /* one sphere query per subscriber (identity batch: query i belongs to subscriber slot i) */
    uint32_t* ring_off;        /* update rings: per-cell CSR of (arrival, sender, message index) */
    int64_t* arrival;
    uint32_t* sender;
    uint64_t *index, *channel_msg_index;
    uint32_t n_ring;
} staging;

static void fill_inputs(staging* s, uint32_t n_entities, uint32_t n_subs, uint32_t cells, int tick) {
    /* a real host copies what arrived since the last tick; here: entities on a slowly rotating lattice */
    for (uint32_t i = 0; i < n_entities; i++) {
        s->x[i] = -14000.0 + (double)((i * 37u + (uint32_t)tick * 11u) % 28000u);
        s->z[i] = -14000.0 + (double)((i * 101u + (uint32_t)tick * 7u) % 28000u);
    }
    for (uint32_t j = 0; j < n_subs; j++) {
        s->cx[j] = s->x[j * (n_entities / n_subs)];
        s->cz[j] = s->z[j * (n_entities / n_subs)];
        s->r[j] = 50.0;
    }
    for (uint32_t c = 0; c <= cells; c++) s->ring_off[c] = 0; /* no channel data updates in this sketch */
    s->n_ring = 0;
    memset(s->channel_msg_index, 0, sizeof(uint64_t) * cells);
}

int main(void) {
    const uint32_t n_entities = 100000, n_subs = 10000;
    const int64_t tick_ns = 33000000;
    chd_grid_cfg cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.world_offset_x = cfg.world_offset_z = -15000.0; /* config/spatial_static_benchmark.json */
    cfg.grid_width = cfg.grid_height = 2000.0;
    cfg.grid_cols = cfg.grid_rows = 15;
    cfg.server_cols = cfg.server_rows = 3;
    cfg.channel_id_start = 65536;
    const uint32_t cells = cfg.grid_cols * cfg.grid_rows;

    chd_limits lim;
    chd_default_limits(&cfg, n_entities, n_subs, &lim);
    chd_engine* e = NULL;
    if (chd_create(&cfg, &lim, 0, &e) != CHD_OK) {
        fprintf(stderr, "chd_create: %s\n", chd_last_error(NULL));
        return 2; /* no GPU: there is no CPU fallback */
    }

    staging st[2];
    for (int k = 0; k < 2; k++) {
        st[k].x = chd_alloc_pinned(8ull * n_entities);
        st[k].z = chd_alloc_pinned(8ull * n_entities);
        st[k].cx = chd_alloc_pinned(8ull * n_subs);
        st[k].cz = chd_alloc_pinned(8ull * n_subs);
        st[k].r = chd_alloc_pinned(8ull * n_subs);
        st[k].ring_off = chd_alloc_pinned(4ull * (cells + 1));
        st[k].arrival = chd_alloc_pinned(8);
        st[k].sender = chd_alloc_pinned(4);
        st[k].index = chd_alloc_pinned(8);
        st[k].channel_msg_index = chd_alloc_pinned(8ull * cells);
    }
    uint32_t* conn = malloc(4ull * n_subs);
    for (uint32_t j = 0; j < n_subs; j++) conn[j] = j + 1; /* connection id of subscriber slot j */
    CHECK(chd_set_subscribers(e, conn, n_subs));

    /* two sets of PINNED result buffers: the read-back of tick k (chd_fetch_results_async) overlaps tick k+1 */
    chd_result_buffers rb[2];
    void* hdr[2];
    for (int k = 0; k < 2; k++) {
        memset(&rb[k], 0, sizeof rb[k]);
        rb[k].pair_cap = rb[k].diff_cap = lim.max_pairs;
        rb[k].due_cap = lim.max_due;
        rb[k].pair_off = chd_alloc_pinned(4ull * (n_subs + 1));
        rb[k].pair_channel = chd_alloc_pinned(4ull * rb[k].pair_cap);
        rb[k].pair_interval_ms = chd_alloc_pinned(4ull * rb[k].pair_cap);
        rb[k].new_sub = chd_alloc_pinned(4ull * rb[k].diff_cap);
        rb[k].new_channel = chd_alloc_pinned(4ull * rb[k].diff_cap);
        rb[k].unsub_sub = chd_alloc_pinned(4ull * rb[k].diff_cap);
        rb[k].unsub_channel = chd_alloc_pinned(4ull * rb[k].diff_cap);
        rb[k].due = chd_alloc_pinned(sizeof(chd_due) * (uint64_t)rb[k].due_cap);
        rb[k].handover_cap = n_entities;
        rb[k].handover_entity = chd_alloc_pinned(4ull * n_entities);
        rb[k].handover_src = chd_alloc_pinned(4ull * n_entities);
        rb[k].handover_dst = chd_alloc_pinned(4ull * n_entities);
        /* the cell CSR makes the result lossless: visible(s) = concatenation of sorted_entity[cell_start[c] .. cell_start[c+1]) over
         * the subscriber's pairs */
        rb[k].cell_start = chd_alloc_pinned(4ull * (cells + 1));
        rb[k].entity_cap = n_entities;
        rb[k].sorted_entity = chd_alloc_pinned(4ull * n_entities);
        hdr[k] = chd_alloc_pinned(CHD_FETCH_HEADER_BYTES);
    }
    /* the visible-set delta of each tick rides in the same fetch: per subscriber slot the entities entered and left */
    const uint64_t delta_cap = 8000000; /* entries per list and tick: the first delta enters every visible entry (about 5e6 here) */
    CHECK(chd_reserve_visible_delta(e, delta_cap));
    chd_delta_buffers db[2];
    for (int k = 0; k < 2; k++) {
        db[k].slot_cap = n_subs + 1ull;
        db[k].entity_cap = delta_cap;
        db[k].enter_off = chd_alloc_pinned(8ull * db[k].slot_cap);
        db[k].leave_off = chd_alloc_pinned(8ull * db[k].slot_cap);
        db[k].enter_entity = chd_alloc_pinned(4ull * delta_cap);
        db[k].leave_entity = chd_alloc_pinned(4ull * delta_cap);
    }

#define PREFETCH(s)                                                                                                       \
    do {                                                                                                                  \
        chd_query_batch q_;                                                                                               \
        memset(&q_, 0, sizeof q_);                                                                                        \
        q_.n = n_subs; /* sub == NULL: identity batch; kind == NULL: all sphere */                                        \
        q_.sph_cx = (s)->cx; q_.sph_cz = (s)->cz; q_.sph_r = (s)->r;                                                      \
        CHECK(chd_prefetch_rings(e, (s)->ring_off, (s)->n_ring, (s)->arrival, (s)->sender, (s)->index, (s)->channel_msg_index)); \
        CHECK(chd_prefetch_queries(e, &q_));                                                                              \
        CHECK(chd_prefetch_entities(e, (s)->x, (s)->z, n_entities));                                                      \
    } while (0)

    fill_inputs(&st[0], n_entities, n_subs, cells, 0);
    PREFETCH(&st[0]);
    chd_tick_summary sum;
    chd_delta_counts dc;
    for (int tick = 0; tick < 100; tick++) {
        const int64_t now = (int64_t)(tick + 1) * tick_ns;
        CHECK(chd_adopt_prefetched(e));            /* inputs of this tick were uploaded during the previous one */
        CHECK(chd_begin_interest(e, NULL, now, 1)); /* interest diff + fan-out pass start on the second stream */
        CHECK(chd_tick(e, NULL, now, CHD_TICK_ALL | CHD_TICK_VISIBLE_DELTA, NULL)); /* asynchronous */
        staging* next = &st[(tick + 1) & 1];
        fill_inputs(next, n_entities, n_subs, cells, tick + 1); /* the host collects tick k+1 while tick k runs */
        PREFETCH(next);
        /* returns at once: device-side sizes, pinned targets */
        CHECK(chd_fetch_results_async_delta(e, &rb[tick & 1], &db[tick & 1], hdr[tick & 1]));
        if (tick == 0) continue;
        /* results of tick - 1, while tick runs on the GPU */
        CHECK(chd_fetch_wait_delta(e, &sum, &dc));
        /* apply from rb[(tick - 1) & 1]: sum.n_sub_new x handleSubToChannel(new_sub[i], new_channel[i]), sum.n_unsub x
         * handleUnsubFromChannel, sum.n_due x fanOutDataUpdate(due[i]), sum.n_handover x the orchestration half of Notify;
         * from db[(tick - 1) & 1]: for each slot s < dc.n_slots spawn enter_entity[enter_off[s] .. enter_off[s + 1]) and despawn
         * leave_entity[leave_off[s] .. leave_off[s + 1]) (dc.deltas == 1: exactly this tick's delta) */
        if ((tick - 1) % 25 == 0)
            printf("tick %d: %llu pairs, %llu visible entries, +%u/-%u subscriptions, %u sends, %u handovers, %llu entered / %llu left\n",
                   tick - 1, (unsigned long long)sum.n_pairs, (unsigned long long)sum.n_visible, sum.n_sub_new, sum.n_unsub, sum.n_due,
                   sum.n_handover, (unsigned long long)dc.n_entered, (unsigned long long)dc.n_left);
    }
    CHECK(chd_fetch_wait_delta(e, &sum, &dc)); /* the last tick */
    chd_destroy(e);

    /* The same world without a position mirror on the host: entities are events keyed by id (entity-table mode) and every
     * subscriber follows its pawn, so each tick is  move -> chd_follow_queries(MOVED) -> chd_begin_interest(NULL) -> chd_tick.
     * Only the moved entities go up; the queries are generated on the device for the followers whose pawn moved. */
    lim.max_queries = 2 * n_subs; /* room for the mixed world below: the explicit part's size class + the followers */
    CHECK(chd_create(&cfg, &lim, 0, &e));
    CHECK(chd_set_subscribers(e, conn, n_subs));
    CHECK(chd_entity_table_init(e));
    {
        uint32_t* id = malloc(4ull * n_entities);
        uint32_t* slot = malloc(4ull * n_subs);
        uint32_t* pawn = malloc(4ull * n_subs);
        for (uint32_t i = 0; i < n_entities; i++) id[i] = 3 * i + 1; /* NetGUID-like ids; 0 and 0xFFFFFFFF are reserved */
        for (uint32_t j = 0; j < n_subs; j++) {
            slot[j] = j;
            pawn[j] = id[(uint64_t)j * (n_entities / n_subs)];
        }
        CHECK(chd_spawn_entities(e, id, st[0].x, st[0].z, n_entities, NULL));
        chd_follow_batch fb;
        memset(&fb, 0, sizeof fb);
        fb.n = n_subs; /* kind == NULL: all sphere */
        fb.slot = slot; fb.entity = pawn; fb.sph_r = st[0].r;
        CHECK(chd_follow_bind(e, &fb));
        const uint32_t n_moved = n_entities / 100;
        uint32_t* mid = chd_alloc_pinned(4ull * n_moved);
        for (int tick = 0; tick < 20; tick++) {
            const int64_t now = (int64_t)(tick + 1) * tick_ns;
            for (uint32_t i = 0; i < n_moved; i++) mid[i] = id[((uint64_t)i * 100 + (uint32_t)tick) % n_entities];
            if (tick) CHECK(chd_move_entities(e, mid, st[tick & 1].x, st[tick & 1].z, n_moved)); /* stand-in positions */
            CHECK(chd_follow_queries(e, tick ? CHD_FOLLOW_MOVED : CHD_FOLLOW_ALL));
            CHECK(chd_begin_interest(e, NULL, now, 0));
            CHECK(chd_tick(e, NULL, now, CHD_TICK_BUILD | CHD_TICK_EMIT, &sum));
            /* after CHD_OVF_PAIRS / CHD_OVF_WINDOW in sum.overflow: generate the next batch with CHD_FOLLOW_ALL */
        }
        uint32_t followers = 0, selected = 0;
        CHECK(chd_get_follow(e, NULL, NULL, NULL, NULL, NULL, 0, &followers, &selected));
        printf("followers: %u bound, %u queries generated for the last tick, %llu pairs\n", followers, selected, (unsigned long long)sum.n_pairs);

        /* A mixed world: every 4th connection is a spectator that sends its own UPDATE_SPATIAL_INTEREST each tick (a sphere
         * anywhere, not on a pawn); the others keep following.  The explicit part is prefetched a tick ahead like any batch, and
         * chd_follow_queries_with(.., NULL) merges the adopted part in front of the generated queries: one interest update, one diff
         * and one read-back per tick, pipelined as above. */
        const uint32_t n_x = (n_subs + 3) / 4;
        uint32_t* xslot = malloc(4ull * n_x);
        for (uint32_t j = 0; j < n_x; j++) xslot[j] = 4 * j;
        CHECK(chd_follow_unbind(e, xslot, n_x));
        double* xq = chd_alloc_pinned(2 * 3 * 8ull * n_x); /* two staging sets of cx | cz | r */
#define PREFETCH_EXPLICIT(k, t)                                                                                           \
    do {                                                                                                                  \
        double* q_ = xq + (uint64_t)(k) * 3 * n_x;                                                                        \
        for (uint32_t j = 0; j < n_x; j++) {                                                                             \
            q_[j] = st[0].x[((uint64_t)j * 7 + (uint32_t)(t)) % n_entities]; /* stand-in camera positions */              \
            q_[n_x + j] = st[0].z[((uint64_t)j * 7 + (uint32_t)(t)) % n_entities];                                        \
            q_[2 * n_x + j] = st[0].r[0];                                                                                 \
        }                                                                                                                 \
        chd_query_batch xb_;                                                                                              \
        memset(&xb_, 0, sizeof xb_);                                                                                      \
        xb_.n = n_x; xb_.sub = xslot; /* sub is required: the part names its slots */                                     \
        xb_.sph_cx = q_; xb_.sph_cz = q_ + n_x; xb_.sph_r = q_ + 2 * n_x;                                                 \
        CHECK(chd_prefetch_queries(e, &xb_));                                                                             \
    } while (0)
        PREFETCH_EXPLICIT(0, 0);
        for (int tick = 0; tick < 20; tick++) {
            const int64_t now = (int64_t)(tick + 21) * tick_ns;
            for (uint32_t i = 0; i < n_moved; i++) mid[i] = id[((uint64_t)i * 100 + (uint32_t)tick) % n_entities];
            CHECK(chd_move_entities(e, mid, st[tick & 1].x, st[tick & 1].z, n_moved));
            CHECK(chd_adopt_prefetched(e));                                /* this tick's explicit part */
            CHECK(chd_follow_queries_with(e, CHD_FOLLOW_MOVED, NULL));     /* ... merged with the followers' queries */
            if (tick + 1 < 20) PREFETCH_EXPLICIT((tick + 1) & 1, tick + 1); /* the adopted set is free again: fill the other */
            CHECK(chd_tick(e, NULL, now, CHD_TICK_BUILD | CHD_TICK_EMIT | CHD_TICK_FOLLOW, NULL));
            CHECK(chd_fetch_results_async(e, &rb[tick & 1], hdr[tick & 1]));
            if (tick) CHECK(chd_fetch_wait(e, &sum)); /* tick - 1: statuses [0, n_x) are the spectators', followers from H on */
        }
        CHECK(chd_fetch_wait(e, &sum));
        printf("mixed world: %u spectators, %llu pairs\n", n_x, (unsigned long long)sum.n_pairs);
#undef PREFETCH_EXPLICIT
        chd_free_pinned(xq);
        free(xslot);
        chd_free_pinned(mid);
        free(id); free(slot); free(pawn);
    }
    chd_destroy(e);
    free(conn);
    return 0;
}
