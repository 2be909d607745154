/*
 * chd_gpu_subs.h — explicit subscriptions to spatial channels (libchd_b200.so, same library as chd_gpu.h).
 *
 * channeld has two writers of a connection's spatial subscriptions: handleUpdateSpatialInterest (chd_update_interest) and
 * SubscribeToChannel / UnsubscribeFromChannel (subscription.go:34-125), reached from handleSubToChannel / handleUnsubFromChannel
 * (message.go:488-605).  The second is how a spatial server subscribes to the cells it owns after CreateChannels
 * (message_spatial.go:167-173) and to its border cells (spatial.go:481-590), and how any connection subscribes to a spatial
 * channel by hand with options the interest path cannot express (FanOutDelayMs, SkipSelfUpdateFanOut, SkipFirstFanOut, any
 * interval).  chd_apply_subscriptions applies a batch of those ops to the engine's (subscriber, cell) pairs, on the device.
 *
 * These calls live in a header of their own so that chd_gpu.h, its structs and its entry-point inventory stay exactly as they
 * are; this header has its own inventory, checked by the same rules.  Plain C99; include it instead of (or after) chd_gpu.h.
 *
 * Semantics (channeldorg/channeld @ 61fa8add):
 *   SUB of a new pair       (subscription.go:59-87) starts from the SPATIAL defaults: chd_limits.default_fanout_interval_ms and
 *                           default_fanout_delay_ms, SkipSelfUpdateFanOut = true, SkipFirstFanOut = false; the fields the op
 *                           carries (present) replace them.  Then lastFanOutTime = the channel's time at now_ns (per-channel
 *                           origins: chd_set_channel_start_times) + delay, hadFirstFanOut = SkipFirstFanOut, lastMessageIndex = 0,
 *                           dist = CHD_DIST_EXPLICIT, and the cell's maxFanOutIntervalMs grows to the interval (subscription.go:84-86).
 *   SUB of an existing pair (subscription.go:44-57): a present interval and SkipSelfUpdateFanOut replace the pair's; delay and
 *                           SkipFirstFanOut act at creation only and are ignored.  Fan-out state and dist stay; maxFanOutIntervalMs
 *                           is not raised.
 *   UNSUB                   (subscription.go:104-125) removes the pair; CHD_SUB_NOT_SUBSCRIBED if there is none.
 *   Several ops on one (slot, channel) apply in array order; each status describes the state its op met (SUB, SUB, UNSUB gives
 *   NEW, MERGED, UNSUBSCRIBED).
 *   Rejected ops change nothing: CHD_SUB_ERR_SLOT for a slot that is free (at or above the slot count, or released: connection id
 *   0) or has a removal or migration pending; CHD_SUB_ERR_CHANNEL for a channel id outside this grid.
 *   Capacity is transactional, as for CHD_OVF_PAIRS in the interest update: if the resulting pair total exceeds
 *   chd_limits.max_pairs nothing is applied, every valid op gets CHD_SUB_ERR_CAPACITY, and the next summary carries CHD_OVF_PAIRS
 *   with required_pairs.  The bit stays set until a summary reads it, and the next interest update overwrites required_pairs with
 *   its own total: a host that wants to tell a refused batch from an interest update that overflowed reads out_status (or calls
 *   chd_summary after the batch) before its next tick; otherwise that tick's summary shows CHD_OVF_PAIRS although its own update
 *   was applied.  A batch holds at most max_pairs ops, and the engine at most 2^20 - 1 subscriber slots (the ops are sorted by
 *   slot in two 10-bit radix passes): CHD_ERR_CAPACITY otherwise, nothing applied.
 * Interaction with the interest update: an explicit pair is an ordinary pair.  A later query of its slot diffs against it
 * (message_spatial.go:82-88): a query that misses its cell unsubscribes it (it appears in that update's unsub list); a query
 * that hits it keeps it, with the damping interval and the query's dist, its flags and fan-out state unchanged.
 * chd_remove_subscribers removes explicit pairs too.  So a follower, or any slot that sends a query every tick, loses the
 * explicit subscriptions its query does not cover; the reference does the same.
 * Everything downstream reads the pairs: the fan-out (due list, window classes, payloads, framing), the expanded visible lists,
 * the visible-set deltas, summary.n_pairs, chd_get_pairs and the fetch paths.  The interest diff lists and n_sub_new / n_unsub /
 * n_kept remain the interest update's alone: out_status is how the host learns what the ops did.
 *
 * Call order and pointers: stream-ordered on the engine stream, a stage of its own between ticks; CHD_ERR_STATE (nothing changes)
 * between chd_begin_interest and the chd_tick that joins it.  The arrays of the batch may be host or device memory; they are copied
 * into engine scratch on the engine stream, under the pointer rules of the other batch inputs (chd_gpu.h: pinned host memory
 * makes the copy asynchronous and is reusable after the next synchronising call).  out_status (host or device) == NULL adds no
 * host synchronisation; otherwise the statuses (one CHD_SUB_* per op) are written before the call returns.  Slab engines
 * (chd_set_slab / chd_comm_init) return CHD_ERR_STATE: they apply explicit subscriptions with chd_apply_subscriptions_sharded
 * (chd_gpu_subs_sharded.h).
 */
#ifndef CHD_GPU_SUBS_H
#define CHD_GPU_SUBS_H
#include "chd_gpu.h"
#ifdef __cplusplus
extern "C" {
#endif

enum { CHD_SUBOP_SUB = 0, CHD_SUBOP_UNSUB = 1 };
/* which ChannelSubscriptionOptions fields an op carries (proto optional presence, channeld.proto) */
enum { CHD_SUBOPT_INTERVAL = 1, CHD_SUBOPT_DELAY = 2, CHD_SUBOPT_SKIP_SELF = 4, CHD_SUBOPT_SKIP_FIRST = 8 };

/* SoA, n ops applied in array order */
typedef struct chd_sub_batch {
    uint32_t        n;
    const uint32_t* slot;         /* subscriber slot (connection -> slot, as for queries) */
    const uint32_t* channel_id;   /* spatial channel id */
    const uint8_t*  op;           /* CHD_SUBOP_* (bit 0 is read: set = UNSUB) */
    const uint8_t*  present;      /* CHD_SUBOPT_* mask per op, or NULL = no field present (defaults / no change) */
    const uint32_t* interval_ms;  /* the arrays of fields no op carries may be NULL (a present bit whose array is NULL reads as absent) */
    const int32_t*  delay_ms;
    const uint8_t*  skip_self;
    const uint8_t*  skip_first;
} chd_sub_batch;

enum {
    CHD_SUB_NEW = 0,            /* subscribed (subscription.go:59-87) */
    CHD_SUB_MERGED = 1,         /* already subscribed: options merged (subscription.go:44-57) */
    CHD_SUB_UNSUBSCRIBED = 2,   /* unsubscribed (subscription.go:104-125) */
    CHD_SUB_NOT_SUBSCRIBED = 3, /* UNSUB of a pair that does not exist (subscription.go:110-113) */
    CHD_SUB_ERR_SLOT = 4,       /* free slot, or a removal / migration pending */
    CHD_SUB_ERR_CHANNEL = 5,    /* channel id outside this grid */
    CHD_SUB_ERR_CAPACITY = 6    /* the batch would exceed max_pairs: nothing was applied */
};

/* chd_get_pairs' dist of a pair that no query has produced */
#define CHD_DIST_EXPLICIT 0xFFFFFFFFu

/* Applies the batch at time now_ns.  out_status[n] (may be NULL): one CHD_SUB_* per op. */
chd_status chd_apply_subscriptions(chd_engine* e, const chd_sub_batch* b, int64_t now_ns, uint8_t* out_status);

#ifdef __cplusplus
}
#endif
#endif
