// chd_delta.cuh — visible-set deltas: per subscriber slot, the entities that entered / left its visible set since the engine's
// snapshot (the state at the last successful delta).  Keys are cell indices, C (= cells) for "not in the world"; an entity index
// at or above a state's entity count is absent from that state.
//
// 1. Moves.  Two look-back scans rank the entries of the current cell CSR whose entity was in another cell (or absent) at the
//    snapshot, and the entries of the snapshot's CSR whose entity is in another cell (or absent) now; a scatter turns the ranks
//    into per-cell ARRIVAL and DEPARTURE lists (CSR by cell, entity order inside a cell: stable by construction).
// 2. Per slot s, with P = its snapshot cells and Q = its current cells (both sorted):
//      entered from c in Q \ P: the members of c now whose snapshot cell is not in P
//      entered from c in Q & P: the arrivals of c whose snapshot cell is not in P
//      left from c in P \ Q:    the snapshot members of c whose current cell is not in Q
//      left from c in P & Q:    the departures of c whose current cell is not in Q
//    Every entity comes out once, cells ascending and entities ascending inside a cell: the order of the visible lists, no sort.
//    A count pass, two scans into u64 offsets and a write pass (one warp per slot).
// 3. The snapshot advances (device-side copies) only if both lists fitted.
//
// Id mode (chd_reserve_visible_delta_ids) runs the same kernels with the entity identity moved from the index to the GLOBAL id:
// the cell CSRs hold global ids there (the build sorts d_gid as its values), so the stage first scatters every in-world entity's
// cell into a key array indexed by global id (delta_id_scatter_kernel) and hands that array to the kernels below as `key`.
#pragma once
#include "chd_scan.cuh"
#include "chd_types.cuh"

namespace chd {

constexpr int DELTA_THREADS = 256;

struct DeltaDev {
    uint32_t cells;
    // now: the last build's keys and cell CSR, the current pairs
    const uint32_t* key;
    uint32_t n;  // entity count of the last build
    const uint32_t *cell_start, *sorted;  // [C+2], [in-world entities]
    const uint32_t *pair_off, *pair_cell;
    uint32_t n_slots;
    // the snapshot
    uint32_t *snap_key, *snap_cell_start, *snap_sorted, *snap_pair_off, *snap_pair_cell, *snap_hdr;
    // moves
    const uint32_t *arr_rank, *dep_rank;
    uint32_t *arr, *dep, *arr_start, *dep_start;
    // outputs
    uint32_t *cnt_enter, *cnt_leave;
    uint64_t *enter_off, *leave_off;
    uint32_t *enter, *leave;
    uint64_t enter_cap, leave_cap;
    uint32_t n_out;  // slots the output CSRs cover (>= n_slots and >= the snapshot's slot count)
    uint32_t* overflow;
    const uint32_t* bad_ids;  // id mode: nonzero when this state's ids are unusable (CHD_OVF_DELTA_IDS); nullptr in index mode
};

// position j of the current cell CSR holds an entity that was elsewhere (or absent) at the snapshot.  Every entity of the
// current CSR is below n, except an out-of-range id of an id-mode state that the stage discards (CHD_OVF_DELTA_IDS).
struct DeltaArrivalFlag {
    const uint32_t *sorted, *key, *snap_key, *snap_hdr;
    uint32_t n, cells;
    __device__ __forceinline__ uint64_t operator()(uint64_t j) const {
        const uint32_t e = sorted[j];
        const uint32_t was = e < snap_hdr[0] ? snap_key[e] : cells;
        const uint32_t now = e < n ? key[e] : cells;
        return was != now ? 1u : 0u;
    }
};

// Id mode: gkey[id] = cell of every in-world entity of the last build (own and halo, i < the build's length), gkey cleared to
// 0xFFFFFFFF (absent) before.  An id >= id_space, or an id that two in-world entities hold, sets *bad and CHD_OVF_DELTA_IDS.
__global__ void __launch_bounds__(DELTA_THREADS) delta_id_scatter_kernel(EntityIds ids, const uint32_t* key, uint32_t n, const uint32_t* n_ptr,
                                                                         uint32_t cells, uint32_t* gkey, uint32_t id_space, uint32_t* bad, uint32_t* overflow) {
    const uint32_t m = n_ptr ? min(*n_ptr, n) : n;
    bool err = false;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const uint32_t k = key[i];
        if (k >= cells) continue;  // an own entity outside the world: absent, never a duplicate
        const uint32_t g = ids.at(i);
        if (g >= id_space || atomicExch(&gkey[g], k) != 0xFFFFFFFFu) err = true;
    }
    if (err) {
        atomicOr(bad, 1u);
        atomicOr(overflow, (uint32_t)CHD_OVF_DELTA_IDS);
    }
}

// position j of the snapshot's cell CSR holds an entity that is elsewhere (or absent) now
struct DeltaDepartureFlag {
    const uint32_t *snap_sorted, *snap_key, *key;
    uint32_t n, cells;
    __device__ __forceinline__ uint64_t operator()(uint64_t j) const {
        const uint32_t e = snap_sorted[j];
        const uint32_t now = e < n ? key[e] : cells;
        return now != snap_key[e] ? 1u : 0u;
    }
};

// ranks -> per-cell arrival / departure lists and their CSR offsets
__global__ void __launch_bounds__(DELTA_THREADS) delta_moves_kernel(DeltaDev d, uint32_t n_max) {
    const uint32_t n_now = d.cell_start[d.cells], n_snap = d.snap_cell_start[d.cells];
    const uint32_t span = max(n_max, d.cells + 1);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < span; i += gridDim.x * blockDim.x) {
        if (i < n_now && d.arr_rank[i + 1] != d.arr_rank[i]) d.arr[d.arr_rank[i]] = d.sorted[i];
        if (i < n_snap && d.dep_rank[i + 1] != d.dep_rank[i]) d.dep[d.dep_rank[i]] = d.snap_sorted[i];
        if (i <= d.cells) {
            d.arr_start[i] = d.arr_rank[d.cell_start[i]];
            d.dep_start[i] = d.dep_rank[d.snap_cell_start[i]];
        }
    }
}

__device__ __forceinline__ bool delta_in_sorted(const uint32_t* a, uint32_t lo, uint32_t hi, uint32_t v) {
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1, x = a[mid];
        if (x == v) return true;
        if (x < v) lo = mid + 1;
        else hi = mid;
    }
    return false;
}

// One side of a slot's delta, executed by a whole warp (all loop bounds are warp-uniform).  For each cell c of `from`
// (ascending): the entities of c's list (the moved ones if c is also in `other`, else all of c's members) whose cell in the other
// state (other_key, absent at or above other_n) is not in `other`.  Counts them; with WRITE, stores them from out[pos] on.
template <bool WRITE>
__device__ __forceinline__ uint32_t delta_side(const uint32_t* from, uint32_t fb, uint32_t fe, const uint32_t* other, uint32_t ob, uint32_t oe,
                                               const uint32_t* full_start, const uint32_t* full, const uint32_t* moved_start, const uint32_t* moved,
                                               const uint32_t* other_key, uint32_t other_n, uint32_t* out, uint64_t pos, uint32_t lane) {
    uint32_t count = 0;
    for (uint32_t i = fb; i < fe; i++) {
        const uint32_t c = from[i];
        const bool both = delta_in_sorted(other, ob, oe, c);
        const uint32_t* list = both ? moved : full;
        const uint32_t lb = both ? moved_start[c] : full_start[c], le = both ? moved_start[c + 1] : full_start[c + 1];
        for (uint32_t base = lb; base < le; base += 32) {
            const uint32_t j = base + lane;
            uint32_t ent = 0;
            bool keep = false;
            if (j < le) {
                ent = list[j];
                // absent in the other state: a key no cell list holds
                keep = ent >= other_n || !delta_in_sorted(other, ob, oe, other_key[ent]);
            }
            const uint32_t m = __ballot_sync(0xffffffffu, keep);
            if (WRITE && keep) out[pos + count + __popc(m & ((1u << lane) - 1u))] = ent;
            count += __popc(m);
        }
    }
    return count;
}

// WRITE = false: per-slot counts; WRITE = true: the lists at the scanned offsets, if both fit (else CHD_OVF_DELTA, nothing written)
// and the state's ids were usable (else nothing written: the scatter raised CHD_OVF_DELTA_IDS)
template <bool WRITE>
__global__ void __launch_bounds__(DELTA_THREADS) delta_slots_kernel(DeltaDev d) {
    if (WRITE && (d.enter_off[d.n_out] > d.enter_cap || d.leave_off[d.n_out] > d.leave_cap)) {
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(d.overflow, (uint32_t)CHD_OVF_DELTA);
        return;
    }
    if (WRITE && d.bad_ids && *d.bad_ids) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t snap_n = d.snap_hdr[0], snap_slots = d.snap_hdr[1];
    for (uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < d.n_out; s += nwarps) {
        const uint32_t qb = s < d.n_slots ? d.pair_off[s] : 0, qe = s < d.n_slots ? d.pair_off[s + 1] : 0;
        const uint32_t pb = s < snap_slots ? d.snap_pair_off[s] : 0, pe = s < snap_slots ? d.snap_pair_off[s + 1] : 0;
        const uint32_t ne = delta_side<WRITE>(d.pair_cell, qb, qe, d.snap_pair_cell, pb, pe, d.cell_start, d.sorted, d.arr_start, d.arr, d.snap_key,
                                              snap_n, d.enter, WRITE ? d.enter_off[s] : 0, lane);
        const uint32_t nl = delta_side<WRITE>(d.snap_pair_cell, pb, pe, d.pair_cell, qb, qe, d.snap_cell_start, d.snap_sorted, d.dep_start, d.dep,
                                              d.key, d.n, d.leave, WRITE ? d.leave_off[s] : 0, lane);
        if (!WRITE && lane == 0) {
            d.cnt_enter[s] = ne;
            d.cnt_leave[s] = nl;
        }
    }
}

// the current state becomes the snapshot, unless a list overflowed or its ids were unusable
__global__ void __launch_bounds__(DELTA_THREADS) delta_advance_kernel(DeltaDev d, uint32_t pairs_max) {
    if (d.enter_off[d.n_out] > d.enter_cap || d.leave_off[d.n_out] > d.leave_cap) return;
    if (d.bad_ids && *d.bad_ids) return;
    const uint32_t n_in = d.cell_start[d.cells], n_pairs = d.pair_off[d.n_slots];
    const uint32_t span = max(max(d.n, pairs_max), max(d.cells + 2, d.n_slots + 1));
    const uint32_t first = blockIdx.x * blockDim.x + threadIdx.x;
    for (uint32_t i = first; i < span; i += gridDim.x * blockDim.x) {
        if (i < d.n) d.snap_key[i] = d.key[i];
        if (i < n_in) d.snap_sorted[i] = d.sorted[i];
        if (i < d.cells + 2) d.snap_cell_start[i] = d.cell_start[i];
        if (i <= d.n_slots) d.snap_pair_off[i] = d.pair_off[i];
        if (i < n_pairs) d.snap_pair_cell[i] = d.pair_cell[i];
    }
    if (first == 0) {
        d.snap_hdr[0] = d.n;
        d.snap_hdr[1] = d.n_slots;
    }
}

}  // namespace chd
