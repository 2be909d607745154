/*
 * chd_gpu_subs_sharded.h — explicit subscriptions to spatial channels on X-slabs (libchd_b200.so, same library as chd_gpu.h).
 *
 * A sharded host (chd_set_slab / chd_comm_init) applies SUB_TO_CHANNEL / UNSUB_FROM_CHANNEL on the rank that holds the subscriber
 * slot, to the cells that rank serves: columns [col_lo - halo, col_hi + halo), clipped to the grid.  There the slot's visible
 * lists, its ring replicas and so its fan-out are exact, as they are for the pairs its queries make.  A spatial server whose region
 * plus border spans more than one rank's served columns is hosted with one subscriber slot per (connection, rank), and each op goes
 * to the slot on the rank that owns the cell's column (channeld_b200/sharding.py: route_sub_ops).
 *
 * This call lives in a header of its own so that chd_gpu.h and chd_gpu_subs.h, their structs and their entry-point inventories stay
 * exactly as they are; chd_apply_subscriptions keeps refusing slab engines.  Plain C99; include it after chd_gpu.h (it includes
 * chd_gpu_subs.h).
 *
 * Semantics: those of chd_apply_subscriptions (chd_gpu_subs.h), with these differences.
 *   The engine must be a slab (chd_set_slab or chd_comm_init), in index, id or entity-table mode: CHD_ERR_STATE otherwise, nothing
 *   changes.
 *   A SUB whose channel is a cell of the grid in a column outside the served range gets CHD_SUB_ERR_OUTSIDE_SLAB and changes
 *   nothing.  Precedence: CHD_SUB_ERR_SLOT, then CHD_SUB_ERR_CHANNEL, then CHD_SUB_ERR_OUTSIDE_SLAB.  An UNSUB of any cell of the
 *   grid is accepted: it can only meet a pair that exists.
 *   A pair created here raises the cell's maxFanOutIntervalMs on this rank, as on one GPU.  The ring-limit exchange
 *   (chd_gpu_rings.h) carries that raise to every rank that serves the cell: chd_tick_sharded does it itself before it appends the
 *   updates staged by chd_rings_append; a host that joins chd_set_slab engines itself calls chd_export_ring_limits /
 *   chd_import_ring_limits after its applies and before chd_rings_append.
 * Call order: CHD_ERR_STATE (nothing changes) between chd_begin_interest and the chd_tick that joins it, and on a communicator engine
 * while ring updates are staged (after chd_rings_append, until chd_tick_sharded).  So per tick, on every rank:
 *   1. the chd_tick_sharded that ends tick k;
 *   2. chd_apply_subscriptions_sharded with the ops for the slots the rank holds;
 *   3. chd_rings_append, chd_migrate_out / chd_migrate_in, the follower calls;
 *   4. chd_tick_sharded for tick k+1.
 * A slot with a migration pending gets CHD_SUB_ERR_SLOT.  A pair created in step 2 on a slot that emigrates in step 3 travels in the
 * migration blob with the slot's other pairs, options and fan-out state included.
 */
#ifndef CHD_GPU_SUBS_SHARDED_H
#define CHD_GPU_SUBS_SHARDED_H
#include "chd_gpu_subs.h"
#ifdef __cplusplus
extern "C" {
#endif

enum { CHD_SUB_ERR_OUTSIDE_SLAB = 7 }; /* SUB of a cell in a column this slab does not serve */

/* Applies the batch at time now_ns on a slab engine.  out_status[n] (may be NULL): one CHD_SUB_* per op. */
chd_status chd_apply_subscriptions_sharded(chd_engine* e, const chd_sub_batch* b, int64_t now_ns, uint8_t* out_status);

#ifdef __cplusplus
}
#endif
#endif
