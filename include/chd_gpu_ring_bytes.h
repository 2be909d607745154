/*
 * chd_gpu_ring_bytes.h — wire payloads from device-owned update rings (libchd_b200.so, same library as chd_gpu.h).
 *
 * chd_assemble_payloads / chd_frame_packets build each decision's CHANNEL_DATA_UPDATE entry from the serialized updateMsg of the
 * ring entries its window selects.  With host-owned rings (chd_set_rings) those bytes come from chd_set_payload_bytes, indexed by
 * ring position; device-owned rings (chd_rings_init / chd_rings_append) reorder their entries on the device (evictions, slides,
 * drops), so the host cannot index them.  The calls below keep each update's bytes in the ring beside its entry: they are evicted,
 * slid and dropped with it, and the payload kernels read them in place.
 *
 *   chd_rings_reserve_bytes  turns device rings into byte-carrying rings: a slab of bytes_per_cell bytes per cell, a byte position
 *                            and length per entry slot (8 B per slot) and byte cursors per cell.  Needs chd_rings_init first and
 *                            no append since that init, staged or applied (CHD_ERR_STATE); CHD_ERR_CAPACITY if cells x
 *                            bytes_per_cell cannot be allocated, CHD_ERR_INVALID for bytes_per_cell == 0 (either way the engine
 *                            keeps the reservation it had).  A later chd_rings_init empties the byte slabs and keeps the reservation.
 *   chd_rings_append_bytes   chd_rings_append, with update k carrying bytes[byte_off[k] .. byte_off[k + 1]), its serialized
 *                            updateMsg (empty is legal).  byte_off is a HOST array of n_updates + 1 non-decreasing offsets; bytes
 *                            (host or device memory, byte_off[n_updates] bytes) is copied.  An update longer than bytes_per_cell, or
 *                            decreasing offsets, return CHD_ERR_INVALID and append nothing.  On a communicator engine the bytes are
 *                            staged with the updates and chd_tick_sharded appends them (chd_gpu_rings.h).
 *   chd_get_ring_bytes       the bytes of every live entry, in the entry order of chd_get_rings: byte_off gets n_live + 1 offsets
 *                            (n_live = chd_get_rings' ring_off[cells]), bytes the concatenation, *total its length.  byte_off and
 *                            bytes may be NULL (then only *total); CHD_ERR_CAPACITY when the bytes do not fit cap_bytes.
 *                            Synchronous; for tests and recovery.
 *
 * Per update of L bytes, in order (ChannelData.OnUpdate, data.go:149-173, with fixed capacities):
 *   1. the entry slab, as without bytes: the live entries slide to the slab start when the tail reaches its end, and a full slab
 *      drops its oldest entry (CHD_OVF_RING);
 *   2. the byte slab: while the live bytes + L exceed bytes_per_cell the oldest entry is dropped, metadata and bytes (CHD_OVF_RING:
 *      the same "capacity too small for the reference's unbounded list" as a full entry slab); then, if the byte tail has no room
 *      for L bytes, the live bytes slide to the slab start;
 *   3. msgIndex++, the entry and its bytes are pushed;
 *   4. the 512 rule evicts as without bytes and releases the bytes of the entry it evicts.
 * While no CHD_OVF_RING is raised the entries, msgIndex and evictions are exactly those of rings without bytes.
 *
 * On a byte-carrying engine chd_set_payload_bytes still supplies each channel's full data message, the type URL and the message
 * type, with n_entries == 0 (otherwise CHD_ERR_INVALID); chd_assemble_payloads reads the entries' bytes from the rings.
 *
 * Call order (mode rule 14, DESIGN.md §5): the reserve between chd_rings_init and the first append; a byte-carrying engine refuses
 * chd_rings_append and an engine without the reservation refuses chd_rings_append_bytes (CHD_ERR_STATE).  On device rings
 * chd_assemble_payloads is refused (CHD_ERR_STATE) if an append was applied (or chd_rings_init called) after the last fan-out pass,
 * whose windows it replays; without the reservation it is refused as before.  Per tick:
 *   one engine:  chd_tick -> chd_assemble_payloads / chd_frame_packets -> chd_rings_append_bytes -> the next chd_tick
 *   slabs:       chd_tick_sharded -> assemble / frame -> applies -> chd_rings_append_bytes (staged) -> the next chd_tick_sharded
 * The reserve and the append are refused while a chd_begin_interest is pending (rule 13); while updates are staged, the reserve, a
 * second append and chd_get_ring_bytes are refused (rule 12).  Refused calls change nothing.
 *
 * Plain C99; include it after chd_gpu.h (it includes it).
 */
#ifndef CHD_GPU_RING_BYTES_H
#define CHD_GPU_RING_BYTES_H
#include "chd_gpu.h"
#ifdef __cplusplus
extern "C" {
#endif

chd_status chd_rings_reserve_bytes(chd_engine* e, uint32_t bytes_per_cell);
chd_status chd_rings_append_bytes(chd_engine* e, const uint32_t* upd_off, uint32_t n_updates, const int64_t* arrival_ns, const uint32_t* sender_conn_id,
                                  const uint64_t* byte_off, const uint8_t* bytes);
chd_status chd_get_ring_bytes(chd_engine* e, uint64_t* byte_off, uint8_t* bytes, uint64_t cap_bytes, uint64_t* total);

#ifdef __cplusplus
}
#endif
#endif
