// chd_follow.cuh — followers: subscriber slots whose area of interest is centred on an entity (chd_follow_bind).  The device keeps
// one binding per slot and turns the bindings into the tick's query batch (chd_follow_queries) from the positions the build reads,
// so the host neither mirrors positions nor packs and uploads queries.
//
// Generation is ONE single-pass compaction over the slots (compact_lookback_kernel, chd_scan.cuh): the flag functor resolves the
// slot's entity, reads its position, decides selected / not selected / no entity and records that per slot; the sink writes the
// query entry at the follower's rank among the selected ones, so the batch is in ascending slot order.  Reading a position by
// entity is a gather of 16 bytes per follower: latency-bound (not measured in isolation).
#pragma once
#include "chd_scan.cuh"
#include "chd_types.cuh"

namespace chd {

constexpr int FOLLOW_THREADS = 256;
// res[] of a slot that is bound but has no query in the generated batch: FOLLOW_NO_QUERY | CHD_FOLLOW_NOT_SELECTED / _NO_ENTITY /
// _OVERRIDDEN / _OUTSIDE_SLAB (a selected follower's res is its batch entry, below 2^31)
constexpr uint32_t FOLLOW_NO_QUERY = 0x80000000u;

// Where a followed entity's position comes from: the arrays the build reads; in entity-table mode through the id table.
struct FollowEntities {
    const double *__restrict__ px, *__restrict__ pz;
    uint32_t n;  // positions that exist: the entity count, or the table's slot capacity
    const uint64_t* __restrict__ table;  // nullptr: index mode
    uint32_t bits;
    const uint32_t* __restrict__ id_of_slot;
    const double *__restrict__ fx, *__restrict__ fz;  // the table's facings (include/chd_gpu_facing.h), nullptr: no entity has one
};

// The columns a slab serves: its queries may touch cells in columns [col_lo - halo, col_hi + halo) (chd_import_halo brings in no
// other entity).  A follower's centre never reaches the host, so the device decides whether the generated query fits: the union
// over the bound kinds of the column span floor((cx - reach - off_x) / w) .. floor((cx + reach - off_x) / w) (reach = sph_r, box_ex,
// cone_r), in the rounded f64 steps of grid_coord, clipped to the world's columns [0, cols) because samples outside the world are
// skipped.  A bounding box, not the samples: conservative.  lo / hi are -inf / +inf on a side where the served range reaches the
// world's edge.  Only slabs whose served range is not the whole world run it (FollowFlag<_, true>).
struct FollowSlab {
    double off_x, w, fcols, lo, hi;
    __device__ __forceinline__ bool outside(const FollowDev& f, uint64_t s, uint32_t kind, double cx) const {
        double a = INFINITY, b = -INFINITY;
        auto span = [&](double r) {
            a = fmin(a, floor(f64div(f64sub(f64sub(cx, r), off_x), w)));
            b = fmax(b, floor(f64div(f64sub(f64add(cx, r), off_x), w)));
        };
        if (kind & CHD_AOI_SPHERE) span(f.sph_r[s]);
        if (kind & CHD_AOI_BOX) span(f.box_ex[s]);
        if (kind & CHD_AOI_CONE) span(f.cone_r[s]);
        // the clipped span is empty (entirely outside the world, or no finite reach): the query path reports that entry itself
        return b >= 0.0 && a < fcols && a <= b && (a < lo || b >= hi);
    }
};

// A framed follower's query from its entity at (x, z) with facing (fx, fz), not (0, 0): the centre offset along and across the
// unit facing and the cone direction turned by the frame's rotation, each step rounded on its own (include/chd_gpu_facing.h).
struct FramedQuery {
    double cx, cz, dx, dz;
    __device__ __forceinline__ FramedQuery(const FollowFrame& fr, uint64_t s, double x, double z, double fx, double fz) {
        const double m = f64sqrt(f64add(f64mul(fx, fx), f64mul(fz, fz)));
        const double ux = f64div(fx, m), uz = f64div(fz, m);
        const double fwd = fr.off_fwd[s], right = fr.off_right[s], rc = fr.rot_cos[s], rs = fr.rot_sin[s];
        cx = f64sub(f64add(x, f64mul(fwd, ux)), f64mul(right, uz));
        cz = f64add(f64add(z, f64mul(fwd, uz)), f64mul(right, ux));
        dx = f64sub(f64mul(fx, rc), f64mul(fz, rs));
        dz = f64add(f64mul(fx, rs), f64mul(fz, rc));
    }
};

// Merged: the batch has a host part (chd_follow_queries_with), whose entries marked their slots in f.ovr.  The flag reads and
// clears the mark of every slot below the slot count, bound or not, so no mark outlives the generation.  Slab: the served-range
// check runs (a separate instantiation: its f64 divisions would raise the register count of every engine's compaction).
// Frame: some follower has a frame (chd_follow_set_frame).  A framed slot's facing joins the MOVED test, its query is generated
// from the frame and recorded in fr for FollowSink and chd_get_follow_frame.  Engines without frames run the other instantiations.
template <bool Merged, bool Slab, bool Frame = false>
struct FollowFlag {
    FollowDev f;
    FollowEntities ent;
    FollowSlab slab;
    uint32_t mode;
    FollowFrame fr;  // (Frame only)
    __device__ __forceinline__ bool operator()(uint64_t s) const {
        if (Merged && f.ovr[s]) {  // the slot's explicit query wins this tick; the next MOVED generation selects it again
            f.ovr[s] = 0;
            if (f.kind[s]) {
                f.res[s] = FOLLOW_NO_QUERY | (uint32_t)CHD_FOLLOW_OVERRIDDEN;
                f.dirty[s] = 1;
            }
            return false;
        }
        if (!f.kind[s]) return false;
        uint32_t p = f.entity[s];
        if (ent.table) {
            // a despawned slot is parked and may be reused by another id: the cached slot counts only while it still holds this id
            const uint32_t id = p;
            p = f.tslot[s];
            if (p >= ent.n || id == 0u || ent.id_of_slot[p] != id) {
                p = tbl_find(ent.table, ent.bits, id, nullptr);
                f.tslot[s] = p;
            }
        }
        if (p >= ent.n) {  // no such entity: no query, and a respawn counts as moved
            f.res[s] = FOLLOW_NO_QUERY | (uint32_t)CHD_FOLLOW_NO_ENTITY;
            f.dirty[s] = 1;
            return false;
        }
        const double x = ent.px[p], z = ent.pz[p];
        bool moved = __double_as_longlong(x) != __double_as_longlong(f.last_x[s]) || __double_as_longlong(z) != __double_as_longlong(f.last_z[s]);
        const bool framed = Frame && fr.on[s];
        double fx = 0.0, fz = 0.0;  // no facing: zero, or a non-finite component
        if (framed) {
            if (ent.fx) {
                fx = ent.fx[p];
                fz = ent.fz[p];
                if (!isfinite(fx) || !isfinite(fz) || (fx == 0.0 && fz == 0.0)) fx = fz = 0.0;
            }
            moved = moved || __double_as_longlong(fx) != __double_as_longlong(fr.last_fx[s]) || __double_as_longlong(fz) != __double_as_longlong(fr.last_fz[s]);
        }
        if (mode == (uint32_t)CHD_FOLLOW_MOVED && !f.dirty[s] && !moved) {
            f.res[s] = FOLLOW_NO_QUERY | (uint32_t)CHD_FOLLOW_NOT_SELECTED;
            return false;
        }
        double cx = x;
        if (!Frame) {
            if (Slab && slab.outside(f, s, f.kind[s], x)) {  // no query; the centre stays the last generated one, and it counts as moved
                f.res[s] = FOLLOW_NO_QUERY | (uint32_t)CHD_FOLLOW_OUTSIDE_SLAB;
                f.dirty[s] = 1;
                return false;
            }
        } else {
            double cz = z, dx = 0.0, dz = 0.0;
            if (framed) {
                if (fx != 0.0 || fz != 0.0) {
                    const FramedQuery g(fr, s, x, z, fx, fz);
                    cx = g.cx; cz = g.cz; dx = g.dx; dz = g.dz;
                } else {  // no facing: the plain query
                    dx = f.cone_dx[s];
                    dz = f.cone_dz[s];
                }
            }
            if (Slab && slab.outside(f, s, f.kind[s], cx)) {  // (the offset centre)
                f.res[s] = FOLLOW_NO_QUERY | (uint32_t)CHD_FOLLOW_OUTSIDE_SLAB;
                f.dirty[s] = 1;
                return false;
            }
            if (framed) {
                fr.last_fx[s] = fx; fr.last_fz[s] = fz;
                fr.cx[s] = cx; fr.cz[s] = cz; fr.dx[s] = dx; fr.dz[s] = dz;
            }
        }
        f.last_x[s] = x;
        f.last_z[s] = z;
        f.dirty[s] = 0;
        return true;
    }
};

// Merged: the followers' entries start at `base` (the host part's size class H).  Frame: a framed slot's centre and cone direction
// are the ones its flag call recorded in fr.
template <bool Merged, bool Frame = false>
struct FollowSink {
    FollowDev f;
    FollowBatch q;
    uint32_t base;
    FollowFrame fr;  // (Frame only)
    __device__ __forceinline__ void operator()(uint64_t s, uint32_t r) const {
        const uint32_t k = Merged ? base + r : r;
        const uint32_t kind = f.kind[s];
        const bool framed = Frame && fr.on[s];
        const double x = framed ? fr.cx[s] : f.last_x[s], z = framed ? fr.cz[s] : f.last_z[s];  // (written by this thread's flag call)
        q.sub[k] = (uint32_t)s;
        q.kind[k] = (uint8_t)kind;
        if (kind & CHD_AOI_SPHERE) {
            q.sph_cx[k] = x; q.sph_cz[k] = z; q.sph_r[k] = f.sph_r[s];
        }
        if (kind & CHD_AOI_BOX) {
            q.box_cx[k] = x; q.box_cz[k] = z; q.box_ex[k] = f.box_ex[s]; q.box_ez[k] = f.box_ez[s];
        }
        if (kind & CHD_AOI_CONE) {
            q.cone_cx[k] = x; q.cone_cz[k] = z;
            q.cone_dx[k] = framed ? fr.dx[s] : f.cone_dx[s];
            q.cone_dz[k] = framed ? fr.dz[s] : f.cone_dz[s];
            q.cone_angle[k] = f.cone_angle[s]; q.cone_r[k] = f.cone_r[s];
        }
        f.res[s] = k;
    }
    __device__ __forceinline__ void total(uint32_t c) const { *q.n_selected = c; }
};

// chd_get_follow: the bound slots in ascending order with what the last generation did with each of them.
struct FollowBoundFlag {
    const uint8_t* __restrict__ kind;
    __device__ __forceinline__ bool operator()(uint64_t s) const { return kind[s] != 0; }
};
struct FollowReportSink {
    FollowDev f;
    const uint32_t* __restrict__ qstatus;  // statuses of the interest update that consumed the batch
    uint32_t *__restrict__ slot, *__restrict__ entity, *__restrict__ status;
    double *__restrict__ cx, *__restrict__ cz;
    uint32_t* __restrict__ count;
    __device__ __forceinline__ void operator()(uint64_t s, uint32_t k) const {
        const uint32_t r = f.res[s];
        slot[k] = (uint32_t)s;
        entity[k] = f.entity[s];
        status[k] = (r & FOLLOW_NO_QUERY) ? (r & ~FOLLOW_NO_QUERY) : qstatus[r];
        cx[k] = f.last_x[s];
        cz[k] = f.last_z[s];
    }
    __device__ __forceinline__ void total(uint32_t c) const { *count = c; }
};

// chd_get_follow_frame: the framed followers in ascending slot order with the facing, centre and direction of their last query.
struct FollowFramedFlag {
    const uint8_t *__restrict__ kind, *__restrict__ on;
    __device__ __forceinline__ bool operator()(uint64_t s) const { return kind[s] != 0 && on[s] != 0; }
};
struct FollowFrameReportSink {
    FollowFrame fr;
    uint32_t* __restrict__ slot;
    double* __restrict__ out;  // [6][cap]: fx, fz, cx, cz, dx, dz
    uint32_t cap;
    uint32_t* __restrict__ count;
    __device__ __forceinline__ void operator()(uint64_t s, uint32_t k) const {
        slot[k] = (uint32_t)s;
        out[k] = fr.last_fx[s];
        out[(uint64_t)cap + k] = fr.last_fz[s];
        out[2ull * cap + k] = fr.cx[s];
        out[3ull * cap + k] = fr.cz[s];
        out[4ull * cap + k] = fr.dx[s];
        out[5ull * cap + k] = fr.dz[s];
    }
    __device__ __forceinline__ void total(uint32_t c) const { *count = c; }
};

// chd_follow_queries_with: the host part `h` (h.n is not read: the replayed graph must not bake the host count in; it is hdr[0],
// written before the graph) copied into the merged arrays q, then skip entries up to H + B.  Grid-stride over the entries and, when
// the host part has spots, over its spot data.  Only the arrays the host part supplies are copied (kind == NULL: all sphere); an
// entry whose kind needs an array it did not supply is marked in q.missing, and the slot of every entry below the slot count is
// marked for FollowFlag.  The compaction that follows writes the selected followers over the skip entries from H on.
struct FollowMerge {
    QueryDev h;
    const uint32_t* __restrict__ hdr;  // [0] host entries n_h
    uint32_t H, len;                   // size class, H + B
    uint32_t n_slots;
    FollowBatch q;
    uint8_t* __restrict__ ovr;
};
__global__ void __launch_bounds__(FOLLOW_THREADS) follow_merge_kernel(FollowMerge m) {
    const QueryDev& h = m.h;
    const FollowBatch& q = m.q;
    const uint32_t n_h = *m.hdr;
    const uint32_t spots = h.spot_off ? h.spot_off[n_h] : 0u;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= m.len; i += stride) {
        if (i < n_h) {
            const uint32_t sub = h.sub[i], kind = query_kind(h, i);
            q.sub[i] = sub;
            q.kind[i] = (uint8_t)kind;
            q.missing[i] = query_arrays_missing(h, kind);
            if (h.sph_cx) q.sph_cx[i] = h.sph_cx[i];
            if (h.sph_cz) q.sph_cz[i] = h.sph_cz[i];
            if (h.sph_r) q.sph_r[i] = h.sph_r[i];
            if (h.box_cx) q.box_cx[i] = h.box_cx[i];
            if (h.box_cz) q.box_cz[i] = h.box_cz[i];
            if (h.box_ex) q.box_ex[i] = h.box_ex[i];
            if (h.box_ez) q.box_ez[i] = h.box_ez[i];
            if (h.cone_cx) q.cone_cx[i] = h.cone_cx[i];
            if (h.cone_cz) q.cone_cz[i] = h.cone_cz[i];
            if (h.cone_dx) q.cone_dx[i] = h.cone_dx[i];
            if (h.cone_dz) q.cone_dz[i] = h.cone_dz[i];
            if (h.cone_angle) q.cone_angle[i] = h.cone_angle[i];
            if (h.cone_r) q.cone_r[i] = h.cone_r[i];
            if (h.spot_off) {
                q.spot_off[i] = h.spot_off[i];
                q.spot_ndist[i] = h.spot_ndist[i];
            }
            if (sub < m.n_slots) m.ovr[sub] = 1;
        } else {
            if (i < m.len) {
                q.sub[i] = 0xFFFFFFFFu;
                q.kind[i] = 0;
                q.missing[i] = 0;
                if (h.spot_off) q.spot_ndist[i] = 0;
            }
            if (h.spot_off) q.spot_off[i] = spots;
        }
    }
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < spots; k += stride) {
        q.spot_x[k] = h.spot_x[k];
        q.spot_z[k] = h.spot_z[k];
        q.spot_dist[k] = h.spot_dist[k];
    }
}

// chd_follow_bind: scatter m staged bindings (one per slot: the host keeps the last of a slot named twice) into the per-slot state.
// A bound slot starts dirty, with no query generated yet.
struct FollowStage {
    const uint32_t *__restrict__ slot, *__restrict__ entity;
    const uint8_t* __restrict__ kind;
    const double* __restrict__ shape;  // [7][m]: sph_r, box_ex, box_ez, cone_dx, cone_dz, cone_angle, cone_r
};
// frame_on: the frame marks once frames exist (a re-bind makes the slot plain), else nullptr
__global__ void __launch_bounds__(FOLLOW_THREADS) follow_bind_kernel(FollowStage st, uint32_t m, FollowDev f, uint8_t* __restrict__ frame_on) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t s = st.slot[i];
    f.entity[s] = st.entity[i];
    f.kind[s] = st.kind[i];
    f.sph_r[s] = st.shape[i];
    f.box_ex[s] = st.shape[(uint64_t)m + i];
    f.box_ez[s] = st.shape[2ull * m + i];
    f.cone_dx[s] = st.shape[3ull * m + i];
    f.cone_dz[s] = st.shape[4ull * m + i];
    f.cone_angle[s] = st.shape[5ull * m + i];
    f.cone_r[s] = st.shape[6ull * m + i];
    f.last_x[s] = 0.0;
    f.last_z[s] = 0.0;
    f.dirty[s] = 1;
    f.tslot[s] = TBL_NONE;
    f.res[s] = FOLLOW_NO_QUERY | (uint32_t)CHD_FOLLOW_NOT_SELECTED;
    if (frame_on) frame_on[s] = 0;
}

// chd_follow_unbind / chd_remove_subscribers: the listed slots follow nothing (slots beyond the state are ignored); frame_on as
// for follow_bind_kernel
__global__ void __launch_bounds__(FOLLOW_THREADS) follow_unbind_kernel(const uint32_t* __restrict__ slot, uint32_t n, uint32_t n_state, uint8_t* __restrict__ kind,
                                                                       uint8_t* __restrict__ frame_on) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && slot[i] < n_state) {
        kind[slot[i]] = 0;
        if (frame_on) frame_on[slot[i]] = 0;
    }
}

// chd_follow_set_frame: scatter m staged frames (one per slot) into the frame state.  The slot turns dirty, so the next MOVED
// generation selects it, and its read-back is zero until then.
struct FollowFrameStage {
    const uint32_t* __restrict__ slot;
    const double* __restrict__ v;  // [4][m]: off_fwd, off_right, rot_cos, rot_sin
};
__global__ void __launch_bounds__(FOLLOW_THREADS) follow_frame_kernel(FollowFrameStage st, uint32_t m, FollowDev f, FollowFrame fr) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t s = st.slot[i];
    fr.on[s] = 1;
    fr.off_fwd[s] = st.v[i];
    fr.off_right[s] = st.v[(uint64_t)m + i];
    fr.rot_cos[s] = st.v[2ull * m + i];
    fr.rot_sin[s] = st.v[3ull * m + i];
    fr.last_fx[s] = fr.last_fz[s] = 0.0;
    fr.cx[s] = fr.cz[s] = fr.dx[s] = fr.dz[s] = 0.0;
    f.dirty[s] = 1;
}

}  // namespace chd
