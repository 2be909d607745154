/*
 * chd_gpu_rings.h — device-owned update rings on sharded engines (libchd_b200.so, same library as chd_gpu.h).
 *
 * A channel's update buffer (ChannelData.OnUpdate, data.go:149-173) drops its oldest entry once it holds more than 512 and that
 * entry is older than the channel's maxFanOutIntervalMs, a maximum that only grows, each time a subscription with a longer interval
 * is created (subscription.go:84-86).  chd_rings_init / chd_rings_append keep these buffers on the device and read the maximum from
 * the engine's pairs.  On X-slabs the pairs of one cell live on every rank whose subscribers reach it, so each rank knows only its
 * own part of the maximum.  The calls below exchange it: after an exchange every rank serving a cell holds the maximum over all
 * ranks, which is the value one whole-world engine holds, and the replicas of a ring on every rank that serves its cell evict
 * exactly what the whole-world ring evicts.
 *
 * These calls live in a header of their own so that chd_gpu.h, its structs and its entry-point inventory stay exactly as they
 * are; this header has its own inventory, checked by the same rules.  Plain C99; include it instead of (or after) chd_gpu.h.
 *
 * Records are (cell index, maxFanOutIntervalMs) pairs of u32 in DEVICE memory.  A rank serves the cells of columns
 * [col_lo - halo, col_hi + halo).
 *   chd_export_ring_limits  writes a record for every served cell whose maximum rose since it was last exported or imported,
 *                           in cell order, at most cap of them, and marks them exported.  *out_count = the records needed; if that
 *                           exceeds cap the call returns CHD_ERR_CAPACITY and marks nothing (the next export repeats them all).
 *                           out_count == NULL adds no host synchronisation; an export that does not fit then raises CHD_OVF_BORDER
 *                           in the next summary.
 *   chd_import_ring_limits  raises each record's cell to the record's value (records of cells outside the grid are ignored) and
 *                           marks the value exported, so it is never exported again.
 * Both need device rings (chd_rings_init) on a slab (chd_set_slab / chd_comm_init), and are refused while a chd_begin_interest is
 * pending, like the other ring inputs (CHD_ERR_STATE, nothing changes).  Both are stream-ordered on the engine stream.
 * Call order per tick, for hosts that join slabs themselves (chd_export_border / chd_import_halo): after its tick every rank
 * exports; every rank imports every record of every rank, its own included, before its next chd_rings_append.  Every rank passes
 * the same whole-grid update batch to chd_rings_append, so the rings of a served cell are replicas that see the same appends in the
 * same order.  A slab that never calls these evicts by its own maximum, as before.
 *
 * chd_comm_init / chd_tick_sharded with device rings: the exchange happens inside the tick.  chd_comm_init reserves a section of
 * each rank's contribution for the records (a count and up to the widest rank's served-cell count of records: the peer exchange
 * moves the live records, the ncclAllGather fallback the padded section, 8 B per served cell and rank).  Every tick:
 *   chd_rings_append (every rank, the same whole-grid updates; the call only uploads them) ... chd_tick_sharded, which exports on
 *   the engine stream before anything forks (the maxima as of the previous tick's end), imports right after the exchange, appends
 *   the staged updates, and only then starts the interest update, whose new subscriptions raise the maxima for the next tick.
 * One chd_rings_append per tick on a communicator engine: while updates are staged, a second chd_rings_append and chd_get_rings,
 * chd_begin_interest, chd_update_interest and chd_tick return CHD_ERR_STATE and change nothing; the next chd_tick_sharded applies
 * them.  With device rings, chd_tick_sharded is refused (CHD_ERR_STATE) while a chd_begin_interest of the host's is pending.
 */
#ifndef CHD_GPU_RINGS_H
#define CHD_GPU_RINGS_H
#include "chd_gpu.h"
#ifdef __cplusplus
extern "C" {
#endif

chd_status chd_export_ring_limits(chd_engine* e, uint32_t* d_records, uint32_t cap, uint32_t* out_count);
chd_status chd_import_ring_limits(chd_engine* e, const uint32_t* d_records, uint32_t n);

#ifdef __cplusplus
}
#endif
#endif
