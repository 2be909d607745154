// chd_table.cuh — entity-table mode (chd_entity_table_init): entities are events keyed by id (channeld's NetGUID,
// pkg/unreal/message.go:20-203) placed in position slots.  The host keeps the id -> slot map, the free-slot FIFO and the
// quarantine; the device keeps an open-addressing id table that the move kernels resolve ids through, the id of every slot, and a
// flag per slot spawned or despawned since the last cell assignment (those are AddEntity / RemoveEntity, not handovers).
//
// Table entries are id << 32 | slot over 2^bits words: 0 is empty (id 0 is reserved), id 0xFFFFFFFF marks a tombstone (also a
// reserved id, so no lookup ever matches it).  Linear probing; inserts take empty words only, so live + tombstones only grow until
// the host rebuilds the table.
#pragma once
#include "chd_types.cuh"

namespace chd {

constexpr int TBL_THREADS = 256;

// Spawn apply (x != nullptr): insert (id, slot), slot -> id, the position, flag the slot, and once facings exist (pfx != nullptr)
// the facing (fx == nullptr: none).  Rebuild (x == nullptr): insert only.
__global__ void __launch_bounds__(TBL_THREADS) tbl_spawn_kernel(uint64_t* table, uint32_t bits, const uint32_t* __restrict__ id, const uint32_t* __restrict__ slot,
                                                                const double* __restrict__ x, const double* __restrict__ z, uint32_t n, uint32_t* id_of_slot,
                                                                double* px, double* pz, uint8_t* flag, const double* __restrict__ fx = nullptr,
                                                                const double* __restrict__ fz = nullptr, double* pfx = nullptr, double* pfz = nullptr) {
    const uint64_t mask = (1ull << bits) - 1ull;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint64_t w = (uint64_t)id[i] << 32 | slot[i];
        for (uint64_t h = tbl_home(id[i], bits);; h = (h + 1) & mask)
            if (atomicCAS(reinterpret_cast<unsigned long long*>(table + h), (unsigned long long)TBL_EMPTY, (unsigned long long)w) == TBL_EMPTY) break;
        if (!x) continue;
        id_of_slot[slot[i]] = id[i];
        px[slot[i]] = x[i];
        pz[slot[i]] = z[i];
        flag[slot[i]] = 1;
        if (pfx) {
            pfx[slot[i]] = fx ? fx[i] : 0.0;
            pfz[slot[i]] = fx ? fz[i] : 0.0;
        }
    }
}

// Despawn apply: tombstone the entry, clear slot -> id, park the slot (NaN: outside the world), flag it.
__global__ void __launch_bounds__(TBL_THREADS) tbl_despawn_kernel(uint64_t* table, uint32_t bits, const uint32_t* __restrict__ id, const uint32_t* __restrict__ slot,
                                                                  uint32_t n, uint32_t* id_of_slot, double* px, double* pz, uint8_t* flag) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint64_t h = 0;
        if (tbl_find(table, bits, id[i], &h) != TBL_NONE) table[h] = TBL_TOMB;
        id_of_slot[slot[i]] = 0;
        px[slot[i]] = __longlong_as_double(0x7FF8000000000000ll);
        pz[slot[i]] = __longlong_as_double(0x7FF8000000000000ll);
        flag[slot[i]] = 1;
    }
}

__device__ __forceinline__ void tbl_block_count(unsigned long long* dst, uint32_t v) {
    __shared__ uint32_t s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    if (v) atomicAdd(&s, v);
    __syncthreads();
    if (threadIdx.x == 0 && s) atomicAdd(dst, (unsigned long long)s);
}

// Move, pass 1: resolve each id to its slot (TBL_NONE: not live, counted) and elect the LAST move of every slot in array order.
__global__ void __launch_bounds__(TBL_THREADS) tbl_move_resolve_kernel(const uint64_t* __restrict__ table, uint32_t bits, const uint32_t* __restrict__ id, uint32_t n,
                                                                       uint32_t* __restrict__ mslot, uint32_t* winner, unsigned long long* stats) {
    uint32_t unknown = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t s = tbl_find(table, bits, id[i], nullptr);
        mslot[i] = s;
        if (s == TBL_NONE) unknown++;
        else atomicMax(winner + s, i + 1);
    }
    tbl_block_count(stats + 1, unknown);
}

// Move, pass 2: the winner of each slot writes the position (f32 widened exactly, as widen_positions_kernel does) and, with Facing,
// its facing, and clears its election for the next call; the others count as superseded.
template <typename T, bool Facing = false>
__global__ void __launch_bounds__(TBL_THREADS) tbl_move_apply_kernel(const uint32_t* __restrict__ mslot, uint32_t* winner, const T* __restrict__ x,
                                                                     const T* __restrict__ z, uint32_t n, double* px, double* pz, unsigned long long* stats,
                                                                     const T* __restrict__ fx = nullptr, const T* __restrict__ fz = nullptr,
                                                                     double* pfx = nullptr, double* pfz = nullptr) {
    uint32_t applied = 0, superseded = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t s = mslot[i];
        if (s == TBL_NONE) continue;
        if (winner[s] == i + 1) {
            px[s] = (double)x[i];
            pz[s] = (double)z[i];
            if (Facing) {
                pfx[s] = (double)fx[i];
                pfz[s] = (double)fz[i];
            }
            winner[s] = 0;
            applied++;
        } else {
            superseded++;
        }
    }
    tbl_block_count(stats + 0, applied);
    tbl_block_count(stats + 2, superseded);
}

// After a build: sorted_id[i] = id of sorted position i (what the emit kernels and the read-back see); advances the device build
// number.  n_ptr: the build's length lives on the device (own + halo), n is then the capacity.
__global__ void __launch_bounds__(TBL_THREADS) tbl_gather_ids_kernel(const uint32_t* __restrict__ sorted_slot, EntityIds ids, uint32_t n,
                                                                     const uint32_t* __restrict__ n_ptr, uint32_t* __restrict__ sorted_id, uint32_t* build_seq) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *build_seq += 1;
    const uint32_t m = n_ptr ? min(*n_ptr, n) : n;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) sorted_id[i] = ids.at(sorted_slot[i]);
}

// chd_handoff_entities, one compaction (compact_1p): the own in-world slots whose column lies outside this rank's slab, with their
// id, the rank owning that column, their slot and their position (chd_handoff_entities_facing: and their facing).
struct HandoffFlag {
    GridDev g;
    const uint32_t* __restrict__ key;
    __device__ __forceinline__ bool operator()(uint64_t i) const {
        const uint32_t k = key[i];
        if (k >= g.cells) return false;  // (free and despawned slots are parked outside the world)
        const uint32_t col = k % g.cols;
        return col < g.col_lo || col >= g.col_hi;
    }
};
struct HandoffSink {
    GridDev g;
    uint32_t world;
    const uint32_t* __restrict__ key;
    EntityIds ids;
    const double *__restrict__ px, *__restrict__ pz;
    uint32_t *__restrict__ id, *__restrict__ slot, *__restrict__ dst;
    double *__restrict__ x, *__restrict__ z;
    uint32_t* __restrict__ count;
    const double *__restrict__ pfx = nullptr, *__restrict__ pfz = nullptr;  // facings to copy out (nullptr: none)
    double *__restrict__ fx = nullptr, *__restrict__ fz = nullptr;
    __device__ __forceinline__ void operator()(uint64_t i, uint32_t k) const {
        id[k] = ids.at((uint32_t)i);
        slot[k] = (uint32_t)i;
        dst[k] = slab_owner(key[i] % g.cols, g.cols, world);
        x[k] = px[i];
        z[k] = pz[i];
        if (pfx) {
            fx[k] = pfx[i];
            fz[k] = pfz[i];
        }
    }
    __device__ __forceinline__ void total(uint32_t c) const { *count = c; }
};

// Handover list, pass 1: move the slot-valued list aside (tmp = entity | src | dst, each `cap` long) with its length.
__global__ void __launch_bounds__(TBL_THREADS) tbl_handover_stash_kernel(HandoverOut ho, uint32_t* __restrict__ tmp, uint32_t* __restrict__ tmp_n) {
    const uint32_t n = min(*ho.count, ho.cap);
    if (blockIdx.x == 0 && threadIdx.x == 0) *tmp_n = n;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        tmp[i] = ho.entity[i];
        tmp[ho.cap + i] = ho.src_cell[i];
        tmp[2ull * ho.cap + i] = ho.dst_cell[i];
    }
}

// Handover list, pass 2 (count zeroed in between): keep the moved entities that were neither spawned nor despawned since the
// previous assignment, named by id.
__global__ void __launch_bounds__(TBL_THREADS) tbl_handover_ids_kernel(HandoverOut ho, const uint32_t* __restrict__ tmp, const uint32_t* __restrict__ tmp_n,
                                                                       const uint8_t* __restrict__ flag, EntityIds ids) {
    const uint32_t n = *tmp_n, lane = threadIdx.x & 31;
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {  // (warp-uniform trip count)
        const uint32_t i = base + threadIdx.x;
        const uint32_t s = i < n ? tmp[i] : 0;
        const bool keep = i < n && !flag[s];
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        uint32_t at = 0;
        if (lane == 0 && m) at = atomicAdd(ho.count, (uint32_t)__popc(m));
        at = __shfl_sync(0xffffffffu, at, 0) + __popc(m & ((1u << lane) - 1u));
        if (keep) {
            ho.entity[at] = ids.at(s);
            ho.src_cell[at] = tmp[ho.cap + i];
            ho.dst_cell[at] = tmp[2ull * ho.cap + i];
        }
    }
}

// Visible-set delta (after delta_slots_kernel<true>): enter lists name slots of now, leave lists slots of the snapshot; both become
// ids (snapshot ids for leave: a despawned slot's id is gone from id_of_slot).  Only if both lists fitted; then the build number
// the delta measured is published in the counters (a quarantined slot is released once the host has read it).
__global__ void __launch_bounds__(TBL_THREADS) tbl_delta_ids_kernel(const uint64_t* __restrict__ enter_off, const uint64_t* __restrict__ leave_off, uint32_t n_out,
                                                                    uint64_t enter_cap, uint64_t leave_cap, uint32_t* enter, uint32_t* leave, EntityIds ids,
                                                                    const uint32_t* __restrict__ snap_id, const uint32_t* __restrict__ build_seq, uint32_t* ok_build) {
    const uint64_t ne = enter_off[n_out], nl = leave_off[n_out];
    if (ne > enter_cap || nl > leave_cap) return;
    const uint64_t first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (uint64_t)gridDim.x * blockDim.x;
    if (first == 0) *ok_build = *build_seq;
    for (uint64_t j = first; j < ne; j += stride) enter[j] = ids.at(enter[j]);
    for (uint64_t j = first; j < nl; j += stride) leave[j] = snap_id[leave[j]];
}

// ... and, after the translation, the snapshot's ids advance with the snapshot (same condition as delta_advance_kernel)
__global__ void __launch_bounds__(TBL_THREADS) tbl_delta_commit_kernel(const uint64_t* __restrict__ enter_off, const uint64_t* __restrict__ leave_off, uint32_t n_out,
                                                                       uint64_t enter_cap, uint64_t leave_cap, EntityIds ids, uint32_t n, uint32_t* __restrict__ snap_id) {
    if (enter_off[n_out] > enter_cap || leave_off[n_out] > leave_cap) return;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) snap_id[i] = ids.at(i);
}

__global__ void __launch_bounds__(TBL_THREADS) tbl_park_kernel(double* px, double* pz, uint32_t n) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        px[i] = __longlong_as_double(0x7FF8000000000000ll);
        pz[i] = __longlong_as_double(0x7FF8000000000000ll);
    }
}

}  // namespace chd
