/*
 * chd_gpu_facing.h — followers that turn with their entity (libchd_b200.so, same library as chd_gpu.h).
 *
 * A follower (chd_follow_bind) centres its query on its entity's position, with a cone direction fixed at bind time.  These calls
 * give entities a facing, carried by the same events that move them, and give followers a frame: a centre offset along and across
 * the facing, and a cone that looks along the facing (optionally turned by a fixed rotation).  The device generates the offset
 * centres and the directions each tick, so a host whose pawns turn neither re-binds them (chd_follow_bind synchronises with the
 * engine stream) nor packs explicit cone rows for them.
 *
 * These calls live in a header of their own so that chd_gpu.h, its structs and its entry-point inventory stay exactly as they
 * are; this header has its own inventory, checked by the same rules.  Plain C99; include it instead of (or after) chd_gpu.h.
 *
 * Facing (entity-table mode only).  Every live table id has a facing (fx, fz): an f64 pair in channeld's (x, z) plane.  A host
 * derives it from the pawn's yaw as (cos yaw, sin yaw): under the Y <-> Z swap of channeld's UE data (unrealpb extension.go), UE's
 * forward (X, Y) is (x, z).  A facing with both components zero, or with a non-finite component, is NO facing.
 *   chd_spawn_entities_facing(_f32)  spawns with a facing.
 *   chd_move_entities_facing(_f32)   sets position and facing together; the facing comes from the move that wins the last-wins
 *                                    election for the position (the last move of the id in array order).
 *   chd_move_entities(_f32)          keeps the facing.
 *   chd_spawn_entities(_f32)         gives no facing, so a table slot reused by another id never inherits one.
 *   f32 facings widen exactly, as positions do.  The facing storage (16 B per table slot) is allocated by the first call of this
 *   header; before it, every entity has no facing.
 *
 * Frame of a follower.  chd_follow_set_frame gives bound followers off_fwd and off_right (f64) and optionally a fixed rotation of
 * the cone (rot_cos, rot_sin; NULL arrays: the identity).  A frame marks its slot dirty, so the next generation selects it under
 * CHD_FOLLOW_MOVED.  The frame is cleared by chd_follow_bind of the slot (a re-bind makes the slot plain again), chd_follow_unbind,
 * chd_remove_subscribers, chd_set_subscribers and chd_migrate_out (which unbinds; the destination binds and frames the slot again).
 *
 * Generation of a framed follower.  The entity is at (x, z) with facing f.  Without a facing the query is exactly that of a plain
 * follower.  Otherwise, every product, sum, square root and quotient rounded separately in this order (no FMA):
 *     m  = sqrt(fx*fx + fz*fz);   ux = fx / m;   uz = fz / m
 *     cx = (x + off_fwd*ux) - off_right*uz;      cz = (z + off_fwd*uz) + off_right*ux
 *     dx = fx*rot_cos - fz*rot_sin;              dz = fx*rot_sin + fz*rot_cos      (identity: dx = fx, dz = fz up to the sign of a zero)
 * Every kind of the binding is centred at (cx, cz); the cone looks along (dx, dz) (the query path normalises the direction);
 * boxes stay axis-aligned.  The right-hand side (-uz, ux) is UE's +Y, the pawn's right, after the swap: off_right > 0 places the
 * centre to the pawn's right.
 * Under CHD_FOLLOW_MOVED a framed follower is selected when it is dirty, or when its entity's position or facing differs bit for
 * bit from the ones its last query was generated from.  On a slab the served-range check (CHD_FOLLOW_OUTSIDE_SLAB) uses the
 * offset centre.  CHD_FOLLOW_NO_ENTITY, CHD_FOLLOW_OVERRIDDEN, merged batches, CHD_TICK_FOLLOW and chd_tick_sharded behave as for
 * plain followers.  chd_get_follow is unchanged for every follower: its cx / cz stay the followed entity's position.
 *
 * Hand-off on slabs.  chd_handoff_entities_facing is chd_handoff_entities plus each entity's facing (0, 0: none); the receiving
 * rank adopts the entities with chd_spawn_entities_facing, so the tick after a slab crossing is exact.
 *
 * Mode rule 11 (DESIGN.md §5): every call here needs entity-table mode, CHD_ERR_STATE otherwise (index mode's positions come from
 * host snapshots and the prefetch pair; a facing there would be a third pipelined input).  chd_follow_set_frame and
 * chd_get_follow_frame follow rule 9 as well.  Call order and pointers: the event calls as their chd_gpu.h counterparts,
 * chd_follow_set_frame as chd_follow_bind (its host arrays are staged before it returns), chd_get_follow_frame as chd_get_follow.
 */
#ifndef CHD_GPU_FACING_H
#define CHD_GPU_FACING_H
#include "chd_gpu.h"
#ifdef __cplusplus
extern "C" {
#endif

/* SoA host arrays, n frames; a slot named twice takes its last frame.  A frame with a non-finite value: CHD_ERR_INVALID, nothing
 * applied.  The rotation is not normalised: (rot_cos, rot_sin) of length k scales the cone direction by k, which the query path
 * normalises away. */
typedef struct chd_follow_frame_batch {
    uint32_t        n;
    const uint32_t* slot;       /* bound follower slots (CHD_ERR_INVALID, nothing applied, if one follows nothing) */
    const double*   off_fwd;    /* centre offset along the facing (NULL: 0) */
    const double*   off_right;  /* centre offset to the facing's right (NULL: 0) */
    const double*   rot_cos;    /* cone rotation (rot_cos, rot_sin) relative to the facing; both NULL: the identity (one NULL: CHD_ERR_INVALID) */
    const double*   rot_sin;
} chd_follow_frame_batch;

/* chd_spawn_entities with a facing per event */
chd_status chd_spawn_entities_facing(chd_engine* e, const uint32_t* id, const double* x, const double* z, const double* fx, const double* fz,
                                     uint32_t n, uint8_t* out_status);
chd_status chd_spawn_entities_facing_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, const float* fx, const float* fz,
                                         uint32_t n, uint8_t* out_status);
/* chd_move_entities with a facing per move */
chd_status chd_move_entities_facing(chd_engine* e, const uint32_t* id, const double* x, const double* z, const double* fx, const double* fz,
                                    uint32_t n);
chd_status chd_move_entities_facing_f32(chd_engine* e, const uint32_t* id, const float* x, const float* z, const float* fx, const float* fz,
                                        uint32_t n);
/* chd_handoff_entities with each entity's facing fx[cap], fz[cap] */
chd_status chd_handoff_entities_facing(chd_engine* e, uint32_t* id, uint32_t* dst_rank, double* x, double* z, double* fx, double* fz, uint32_t cap,
                                       uint32_t* count);
/* frames of bound followers */
chd_status chd_follow_set_frame(chd_engine* e, const chd_follow_frame_batch* b);
/* Every framed follower in ascending slot order: the facing its last query used (0, 0: none), that query's centre and its cone
 * direction (without a facing: the entity's position and the bound cone direction).  count: framed followers (may exceed cap). */
chd_status chd_get_follow_frame(chd_engine* e, uint32_t* slot, double* fx, double* fz, double* cx, double* cz, double* dx, double* dz, uint32_t cap,
                                uint32_t* count);

#ifdef __cplusplus
}
#endif
#endif
